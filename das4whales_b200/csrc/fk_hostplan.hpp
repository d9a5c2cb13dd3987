// fk_hostplan.hpp -- host-only planning of the f-k filter (tile width, T1 x T2 split of the
// time axis, twiddle / digit-reversal / taper tables).  Shared by d4w_fk.cu (which uploads
// the tables) and tests/host_emul (which runs the kernel bodies on the CPU).
#pragma once
#include <cstdlib>
#include "fft_plan.hpp"

namespace d4w {

struct FkHostPlan {
    int nx = 0, ns = 0;
    int t1 = 1, t2 = 0, nc = 1, nc_shift = 0, fstride = 0, aligned = 0;
    int dual = 0, npair = 0, npair_shift = 0, aligned16 = 0, tma = 0, col_max_radix = 0;
    int row_dual = 0;
    int row_fused = 0;                // k_row_mid_fused: first stage from global memory, last stage + mask in registers
    // two-level column transform (nx = x1 * x2), see fk_kernels.cuh
    int two_level = 0, x1 = 0, x2 = 0, planes = 0, np2 = 0, fstride2 = 0;
    FftPlan plb{};
    std::vector<float2> tw_x2;
    std::vector<int> pos_x2;        // k2 -> position after the level-B forward transform
    size_t colb_smem = 0;
    int colb_threads = 128;
    int pipe = 0, pipe_lag = 2, pipe_cq = 80;   // single-launch pipelined level A+B (V ring resident in L2)
    int chunk_pairs = 0;              // sample pairs per level-A/level-B launch pair (V chunk sized to stay in L2)
    int fused_ra = 0, fused_rb = 0;   // level B as a fused two-stage transform (X2 = ra * rb) when both radices are in {16, 20, 25}
    int fused3 = 0, r3[3] = {0, 0, 0};   // X1 = 10 with a three-stage small-radix level B (k_col3_pipe), opt-in: D4W_COL_PIPE3=1
    // chirp-z column transform (channel counts with a prime factor > 61): colpl is the length-czt_m plan, tw_col its
    // twiddles, and the single-level kernels' slot positions are natural wavenumbers (pos2k = k2pos = identity)
    int czt = 0, czt_m = 0;
    std::vector<float2> czt_chirp;    // c[n] = exp(-i pi (n^2 mod 2 nx) / nx), n < nx
    std::vector<float2> czt_bhat;     // FFT_M(conj c, wrapped) / M in the M plan's transform order
    FftPlan colpl{}, rowpl{};
    std::vector<float2> tw_col, tw_row, twT;
    std::vector<int> pos2k, k2pos, pos2k_row;
    std::vector<int> pos2k_row_tab;   // frequency of each entry of P3's mask table (table order depends on row_fused)
    std::vector<float> taper;
    size_t col_smem = 0, row_smem = 0;
};

inline int env_int(const char* name, int dflt) {
    const char* s = std::getenv(name);
    return (s && *s) ? std::atoi(s) : dflt;
}

// scipy.signal.windows.tukey(M, alpha) (sym=True): the window dsp.taper_data applies (dsp.py:721)
inline std::vector<float> tukey_window(int m, double alpha) {
    std::vector<float> w((size_t)std::max(m, 0), 1.0f);
    if (m <= 1 || alpha <= 0) return w;
    const double pi = 3.14159265358979323846;
    if (alpha >= 1.0) {
        for (int n = 0; n < m; ++n) w[n] = (float)(0.5 - 0.5 * std::cos(2.0 * pi * n / (m - 1)));
        return w;
    }
    const int width = (int)std::floor(alpha * (m - 1) / 2.0);
    for (int n = 0; n <= width; ++n)
        w[n] = (float)(0.5 * (1.0 + std::cos(pi * (-1.0 + 2.0 * n / alpha / (m - 1)))));
    for (int n = m - width - 1; n < m; ++n)
        w[n] = (float)(0.5 * (1.0 + std::cos(pi * (-2.0 / alpha + 1.0 + 2.0 * n / alpha / (m - 1)))));
    return w;
}

// Chirp-z (Bluestein) channel transform for an nx with a prime factor > 61:
//   X[k] = c[k] * sum_n (x[n] c[n]) conj(c[k - n]),   c[n] = exp(-i pi n^2 / nx),
// the sum being a circular convolution of length M >= 2 nx - 1 (FFT_M -> x B^ -> IFFT_M).  One M-point complex column
// per time-sample pair must fit the single-level column budget `col_budget` (200 KB on an H100: M <= 25 600, so
// nx <= 12 800).
// Largest channel count with a prime factor > 61 whose chirp-z column fits `col_budget` bytes.
inline int czt_max_channels(size_t col_budget) {
    int mmax = (int)std::min<size_t>(col_budget / sizeof(float2), 1 << 30);
    while (mmax > 1 && next_5smooth(mmax) != mmax) --mmax;          // largest 5-smooth M that fits
    return (mmax + 1) / 2;                                          // every nx with 2 nx - 1 <= M gets an M' <= M
}

// Chirp and kernel-spectrum tables of a length-n chirp-z transform over an m-point convolution (m >= 2 n - 1):
// chirp[j] = c[j] = exp(-i pi (j^2 mod 2n) / n) for j < n (exact 64-bit reduction of the phase), and
// bhat[p] = FFT_m(conj c, wrapped)[tab2freq[p]] / m, computed in double and rounded to fp32 once.  tab2freq maps each
// table entry to its frequency, i.e. the order in which the consuming kernel reads the spectrum.
inline void czt_tables(int n, int m, const std::vector<int>& tab2freq, std::vector<float2>& chirp, std::vector<float2>& bhat) {
    const double pi = 3.14159265358979323846;
    const long long two_n = 2LL * n;
    auto phase = [&](long long j) { return pi * (double)((j * j) % two_n) / (double)n; };   // exact integer reduction
    chirp.resize((size_t)n);
    for (int j = 0; j < n; ++j) { const double a = phase(j); chirp[j] = make_float2((float)std::cos(a), (float)(-std::sin(a))); }
    std::vector<double> re((size_t)m, 0.0), im((size_t)m, 0.0);      // b = conj(c), wrapped: b[j] and b[M - j] = b[-j]
    for (int j = 0; j < n; ++j) {
        const double a = phase(j);
        re[j] = std::cos(a); im[j] = std::sin(a);
        if (j > 0) { re[m - j] = re[j]; im[m - j] = im[j]; }
    }
    dft_5smooth_double(re, im);
    bhat.resize((size_t)m);
    for (int p = 0; p < m; ++p) bhat[p] = make_float2((float)(re[tab2freq[p]] / m), (float)(im[tab2freq[p]] / m));
}

// Fills the column fields of hp for the chirp-z transform; returns 0, or 1 with err set.
inline int plan_czt_columns(int nx, size_t col_budget, FkHostPlan& hp, std::string& err) {
    const int m = next_5smooth(2 * nx - 1);
    if ((size_t)m * sizeof(float2) > col_budget) {
        err = "channel axis: " + std::to_string(nx) + " channels has a prime factor > 61, and its chirp-z column transform (" +
              std::to_string(m) + " points) does not fit one SM's column budget: such channel counts are limited to " +
              std::to_string(czt_max_channels(col_budget)) + "; filter a channel sub-range or decimate the channel axis";
        return 1;
    }
    std::string e2;
    FftPlan pl;
    if (!make_plan(m, 25, pl, e2, 256, 16)) { err = "channel axis (chirp-z length " + std::to_string(m) + "): " + e2; return 1; }
    int nc = 8;                                                      // columns per tile, odd stride between them
    while (nc > 1 && (size_t)nc * (m | 1) * sizeof(float2) > col_budget) nc >>= 1;
    hp.czt = 1; hp.czt_m = m; hp.colpl = pl;
    hp.nc = nc; hp.nc_shift = (nc == 1) ? 0 : (nc == 2) ? 1 : (nc == 4) ? 2 : 3;
    hp.fstride = nc == 1 ? m : (m | 1); hp.col_smem = (size_t)nc * hp.fstride * sizeof(float2);
    hp.dual = 0; hp.npair = 0; hp.npair_shift = 0; hp.tma = 0;
    czt_tables(nx, m, make_pos2freq(pl), hp.czt_chirp, hp.czt_bhat);
    return 0;
}

inline const std::vector<int>& split_radices() {
    static const std::vector<int> r = {1, 2, 3, 4, 5, 6, 8, 10, 12, 15, 16, 20, 25};
    return r;
}

// returns 0 on success; 1 = unsupported shape (err says why)
// row_fused_default: whether the middle row pass uses k_row_mid_fused unless D4W_ROW_FUSED says otherwise
inline int build_fk_hostplan(int nx, int ns, size_t smem_cap, FkHostPlan& hp, std::string& err, bool allow_row_dual = true,
                             int row_fused_default = 0) {
    hp.nx = nx; hp.ns = ns;
    const int col_maxr = env_int("D4W_COL_MAX_RADIX", 25);
    const int row_maxr = env_int("D4W_ROW_MAX_RADIX", 25);
    std::string e2;
    int nc = 8;
    const size_t col_budget = std::min<size_t>(smem_cap, 200 * 1024);
    while (nc > 1 && (size_t)nc * (nx + 1) * sizeof(float2) > col_budget) nc >>= 1;
    if ((size_t)nc * (nx + 1) * sizeof(float2) > smem_cap) {
        err = "channel axis too long (" + std::to_string(nx) + " channels): one column of the wavenumber transform must fit one SM's "
              "shared memory (about 28 000 channels, " + std::to_string(czt_max_channels(col_budget)) +
              " when the count has a prime factor > 61); filter a channel sub-range or decimate the channel axis";
        return 1;
    }
    const int forced_nc = env_int("D4W_COL_NC", 0);
    if ((forced_nc == 1 || forced_nc == 2 || forced_nc == 4 || forced_nc == 8) &&
        (size_t)forced_nc * (nx + 1) * sizeof(float2) <= smem_cap) nc = forced_nc;
    hp.nc = nc;
    hp.nc_shift = (nc == 1) ? 0 : (nc == 2) ? 1 : (nc == 4) ? 2 : 3;
    hp.fstride = nx | 1;
    hp.aligned = (ns % 2 == 0) ? 1 : 0;
    hp.col_smem = (size_t)nc * hp.fstride * sizeof(float2);
    // dual-lane (f32x2) column kernels: two complex columns per thread, radix <= 16 (register budget)
    hp.dual = (nc >= 2 && env_int("D4W_COL_DUAL", 1)) ? 1 : 0;
    hp.npair = nc / 2;
    hp.npair_shift = (hp.npair <= 1) ? 0 : (hp.npair == 2) ? 1 : 2;
    hp.aligned16 = (ns % 4 == 0) ? 1 : 0;
    // TMA path: one dual column per tile, rows 16-byte aligned; tile padded to whole 256-row boxes
    hp.tma = (hp.dual && hp.npair == 1 && hp.aligned16 && env_int("D4W_COL_TMA", 1) &&
              (size_t)((nx + 255) / 256 * 256) * 16 <= smem_cap - 1024) ? 1 : 0;
    if (hp.tma) { hp.fstride = (nx + 255) / 256 * 256; hp.col_smem = (size_t)hp.fstride * 16; }
    const char* col_spec = std::getenv("D4W_COL_PLAN");
    if (!(col_spec && *col_spec && make_plan_from_string(nx, col_spec, hp.colpl)) &&
        !make_plan(nx, hp.dual ? std::min(col_maxr, env_int("D4W_DUAL_MAX_RADIX", 25)) : col_maxr, hp.colpl, e2, 256, hp.dual ? 8 : 16)) {
        if (!has_prime_factor_above_61(nx)) { err = "channel axis: " + e2; return 1; }
        if (plan_czt_columns(nx, col_budget, hp, err)) return 1;       // single-level chirp-z column kernels only
    }

    // time axis = T1 (registers) x T2 (shared memory).  Dual-lane row kernel (default): T2 <= 6144 keeps the
    // 16-byte-element tile under 96 KB -> two CTAs per SM; scalar kernel: T2 <= 10240 (16384 when T1 == 1).
    int t1 = 0;
    const int forced_t1 = env_int("D4W_T1", 0);
    hp.row_dual = (allow_row_dual && env_int("D4W_ROW_DUAL", 0)) ? 1 : 0;   // measured: scalar 16x25x25 + cp.async is faster (1.69 vs 1.91 ms)
    const int row_maxr_eff = hp.row_dual ? std::max(row_maxr, 25) : row_maxr;
    for (int cand : split_radices()) {
        if (forced_t1 > 0 && cand != forced_t1) continue;
        if (ns % cand) continue;
        const int t2 = ns / cand;
        const int limit = hp.row_dual ? 6144 : ((cand == 1) ? 16384 : 10240);
        if (forced_t1 == 0 && t2 > limit) continue;
        if ((size_t)t2 * (hp.row_dual ? 16 : 8) > smem_cap - 1024) continue;
        FftPlan tmp;
        if (!make_plan(t2, row_maxr_eff, tmp, e2, hp.row_dual ? 128 : 256, hp.row_dual ? 8 : 16)) continue;
        t1 = cand; hp.rowpl = tmp;
        break;
    }
    if (t1 == 0 && hp.row_dual) {     // no split fits the dual tile: fall back to the scalar row kernel's limits
        hp.row_dual = 0;
        for (int cand : split_radices()) {
            if (forced_t1 > 0 && cand != forced_t1) continue;
            if (ns % cand) continue;
            const int t2 = ns / cand;
            const int limit = (cand == 1) ? 16384 : 10240;
            if (forced_t1 == 0 && t2 > limit) continue;
            if ((size_t)t2 * sizeof(float2) > smem_cap) continue;
            FftPlan tmp;
            if (!make_plan(t2, row_maxr, tmp, e2)) continue;
            t1 = cand; hp.rowpl = tmp;
            break;
        }
    }
    if (t1 == 0) {
        err = "time axis length " + std::to_string(ns) +
              " has no supported split (needs ns = T1*T2 with T1 <= 25, T2 <= 6144 (10240 scalar) and prime factors <= 61)";
        return 1;
    }
    // ---- small-radix variant: X1 = 10 in registers, X2 = R0*R1*R2 with radices <= 10 (three-stage level B), single pipelined launch
    if (!hp.czt && env_int("D4W_COL_TWO_LEVEL", 1) && env_int("D4W_COL_PIPE3", 0) && ns % 4 == 0 && nx % 10 == 0) {
        const int x2 = nx / 10;
        static const int cand[][3] = {{10, 10, 10}, {5, 5, 4}};
        for (auto& c : cand) {
            if (c[0] * c[1] * c[2] != x2) continue;
            FftPlan tmp;
            const std::string spec = std::to_string(c[0]) + "," + std::to_string(c[1]) + "," + std::to_string(c[2]);
            if (!make_plan_from_string(x2, spec.c_str(), tmp)) continue;
            int np = env_int("D4W_PIPE3_NP", 4);
            if (np != 1 && np != 2 && np != 4 && np != 8) np = 4;
            int threads = env_int("D4W_PIPE3_THREADS", 200);
            int cq = env_int("D4W_PIPE3_CQ", 50);
            if (threads < 32 || threads > 224 || cq < 2 || threads % cq || (2 * cq) % np) { threads = 200; cq = 50; np = 4; }
            hp.two_level = 1; hp.x1 = 10; hp.x2 = x2; hp.planes = 6; hp.np2 = np; hp.fstride2 = x2 | 1;
            hp.plb = tmp; hp.colb_smem = (size_t)np * hp.fstride2 * 16;
            hp.fused3 = 1; hp.r3[0] = c[0]; hp.r3[1] = c[1]; hp.r3[2] = c[2];
            hp.pipe = 1; hp.pipe_cq = cq; hp.chunk_pairs = std::min(2 * cq, ns / 2);
            hp.pipe_lag = std::min(256, std::max(1, env_int("D4W_PIPE_LAG", 2)));
            hp.colb_threads = threads;
            hp.tw_x2 = make_twiddles(x2);
            auto p2k = make_pos2freq(tmp);
            hp.pos_x2.assign((size_t)x2, 0);
            for (int p = 0; p < x2; ++p) hp.pos_x2[p2k[p]] = p;
            break;
        }
    }
    // ---- two-level column split: X1 in registers (largest of 25, 20, 16), X2-point smem FFT
    if (!hp.czt && !hp.fused3 && env_int("D4W_COL_TWO_LEVEL", 1) && ns % 4 == 0) {
        const int forced_x1 = env_int("D4W_COL_X1", 0);
        for (int cand : {25, 20, 16}) {
            if (forced_x1 && cand != forced_x1) continue;
            if (nx % cand) continue;
            const int x2 = nx / cand;
            if (x2 < 8 || x2 > 1024) continue;
            FftPlan tmp;
            const char* bspec = std::getenv("D4W_COLB_PLAN");
            if (!(bspec && *bspec && make_plan_from_string(x2, bspec, tmp)) && !make_plan(x2, 25, tmp, e2, 160, 8)) continue;
            int np = 8;
            while (np > 1 && (size_t)np * (x2 | 1) * 16 > 56 * 1024) np >>= 1;
            if ((size_t)np * (x2 | 1) * 16 > 100 * 1024) continue;
            hp.two_level = 1; hp.x1 = cand; hp.x2 = x2; hp.planes = cand / 2 + 1; hp.np2 = np; hp.fstride2 = x2 | 1;
            hp.plb = tmp; hp.colb_smem = (size_t)np * hp.fstride2 * 16;
            int bmax = 1;                                    // most butterflies any stage has per tile
            for (int st = 0; st < tmp.nstages; ++st) bmax = std::max(bmax, (x2 / tmp.radix[st]) * np);
            hp.colb_threads = std::min(160, std::max(64, (bmax + 31) / 32 * 32));
            hp.colb_threads = std::min(160, std::max(32, env_int("D4W_COLB_THREADS", hp.colb_threads)));
            {
                // V chunk = planes * x2 * pairs * 16 B; keep it well inside the H100's 50 MB L2 (D4W_COL_CHUNK_MB = 0: one chunk)
                const int mb = env_int("D4W_COL_CHUNK_MB", 16);
                const long long per_pair = (long long)hp.planes * x2 * 16;
                long long pairs = mb > 0 ? (long long)mb * 1000000 / per_pair / 256 * 256 : (long long)ns / 2;
                pairs = std::max<long long>(pairs, 256);
                const int forced = env_int("D4W_COL_CHUNK_PAIRS", 0);           // test knob; multiple of 8
                if (forced > 0) pairs = std::max(8, forced / 8 * 8);
                hp.chunk_pairs = (int)std::min<long long>(pairs, ns / 2);
            }
            if (env_int("D4W_COLB_FUSED", 1)) {
                // prefer the balanced split (equal item counts in both stages), else the plan's own two radices
                const int forced_ra = env_int("D4W_COLB_RA", 0);
                for (int ra : {20, 16, 25}) {
                    if (forced_ra && ra != forced_ra) continue;
                    if (x2 % ra) continue;
                    const int rb = x2 / ra;
                    if (rb != 16 && rb != 20 && rb != 25) continue;
                    hp.fused_ra = ra; hp.fused_rb = rb;
                    break;
                }
                if (hp.fused_ra) {
                    const int items = std::max(hp.fused_ra, hp.fused_rb) * np;
                    hp.colb_threads = std::min(160, std::max(64, (items + 31) / 32 * 32));
                    hp.colb_threads = std::min(160, std::max(32, env_int("D4W_COLB_THREADS", hp.colb_threads)));
                }
            }
            // pipelined single launch: needs the fused level B with (ra, rb) in {(20,20), (16,25)} and 8-pair tiles
            if (env_int("D4W_COL_PIPE", 1) && hp.fused_ra && np == 8 &&
                ((hp.fused_ra == 20 && hp.fused_rb == 20) || (hp.fused_ra == 16 && hp.fused_rb == 25))) {
                // strip width in quads; 160 threads = cq x rpc.  40 keeps the 4-chunk V ring (13 planes x 400 x 80 pairs x 16 B
                // = 6.7 MB per chunk, 27 MB in all at 10 000 channels) inside the H100's 50 MB L2; 80 (13.3 MB chunks, a 53 MB
                // ring) measured 10 % slower
                int cq = env_int("D4W_PIPE_CQ", 40);
                if (cq < 4 || 160 % cq || (2 * cq) % np) cq = 40;
                hp.pipe = 1; hp.pipe_cq = cq; hp.chunk_pairs = 2 * cq;
                hp.pipe_lag = std::min(256, std::max(1, env_int("D4W_PIPE_LAG", 2)));
                hp.colb_threads = 160;
            }
            hp.tw_x2 = make_twiddles(x2);
            auto p2k = make_pos2freq(tmp);
            hp.pos_x2.assign((size_t)x2, 0);
            for (int p = 0; p < x2; ++p) hp.pos_x2[p2k[p]] = p;
            break;
        }
    }
    for (int st = 0; st < hp.colpl.nstages; ++st) hp.col_max_radix = std::max(hp.col_max_radix, hp.colpl.radix[st]);
    hp.t1 = t1; hp.t2 = ns / t1;
    hp.row_smem = (size_t)hp.t2 * (hp.row_dual ? 16 : sizeof(float2));
    hp.tw_col = make_twiddles(hp.czt ? hp.czt_m : nx);
    hp.tw_row = make_twiddles(hp.t2);
    hp.twT.resize((size_t)hp.t2);
    for (int j = 0; j < hp.t2; ++j) {
        const double a = 6.283185307179586476925286766559 * (double)j / (double)ns;
        hp.twT[j] = make_float2((float)std::cos(a), (float)(-std::sin(a)));
    }
    if (hp.czt) {                     // the chirp-z column leaves wavenumbers in natural order
        hp.pos2k.resize((size_t)nx);
        for (int p = 0; p < nx; ++p) hp.pos2k[p] = p;
    } else {
        hp.pos2k = make_pos2freq(hp.colpl);
    }
    hp.k2pos.assign((size_t)nx, 0);
    for (int p = 0; p < nx; ++p) hp.k2pos[hp.pos2k[p]] = p;
    hp.pos2k_row = make_pos2freq(hp.rowpl);
    hp.pos2k_row_tab = hp.pos2k_row;
    {
        const int nst = hp.rowpl.nstages;
        auto inreg = [](int r) { for (int q : inreg_radices()) if (q == r) return true; return false; };
        // f-k filter (default 0): on sm_90 k_row_mid_fused spills at its 128-register cap, and P3 ran 8.6 ms against 2.3 ms
        // for k_row_mid (H100); the Hilbert plan passes 1, see d4w_row_plan_create
        if (!hp.row_dual && env_int("D4W_ROW_FUSED", row_fused_default) && nst >= 2 && inreg(hp.rowpl.radix[0]) && inreg(hp.rowpl.radix[nst - 1])) {
            hp.row_fused = 1;
            const int rl = hp.rowpl.radix[nst - 1], G = hp.t2 / rl;
            for (int m = 0; m < rl; ++m)
                for (int j = 0; j < G; ++j) hp.pos2k_row_tab[(size_t)m * G + j] = hp.pos2k_row[(size_t)j * rl + m];
        }
    }
    hp.taper = tukey_window(ns, 0.03);
    return 0;
}

// ---- Hilbert rows of any length: chirp-z (Bluestein) row transform -------------------------------------------------
// A row length n that the time-axis planner rejects is transformed as a circular convolution of length m: the smallest
// 2^a 3^b 5^c >= 2 n - 1 that build_fk_hostplan(1, m) accepts.  m <= 25 x 10 240 = 256 000, so n <= 128 000.
constexpr int kHilbertMaxSamples = 128000;

struct RowCztPlan {
    int n = 0, m = 0;
    int fused = 0;                    // split rows: middle pass by k_row_mid_fused (tables in its order)
    FkHostPlan hp;                    // the length-m row plan (t1, t2, rowpl, twiddles, table orders)
    std::vector<float2> chirp;        // c[t], t < n
    std::vector<float2> bhat;         // FFT_m(conj c, wrapped) / m in the middle pass's table order
};

// returns 0, or 1 with err set (n above kHilbertMaxSamples)
inline int plan_czt_rows(int n, size_t smem_cap, RowCztPlan& rp, std::string& err, int row_fused_default = 1) {
    if (n < 1 || n > kHilbertMaxSamples) {
        err = "row length " + std::to_string(n) + " has no mixed-radix split, and chirp-z rows are limited to " +
              std::to_string(kHilbertMaxSamples) + " samples; crop the record";
        return 1;
    }
    std::string e2;
    int m = next_5smooth(2 * n - 1);
    while (build_fk_hostplan(1, m, smem_cap, rp.hp, e2, /*allow_row_dual=*/false, row_fused_default)) {
        m = next_5smooth(m + 1);
        if (m > 25 * 10240) { err = "row length " + std::to_string(n) + ": no chirp-z length fits the row engine"; return 1; }
        rp.hp = FkHostPlan();
    }
    const FkHostPlan& hp = rp.hp;
    rp.n = n; rp.m = m;
    rp.fused = (hp.t1 > 1 && hp.row_fused) ? 1 : 0;
    const std::vector<int>& order = rp.fused ? hp.pos2k_row_tab : hp.pos2k_row;
    std::vector<int> tab2freq((size_t)m);
    for (int kt1 = 0; kt1 < hp.t1; ++kt1)
        for (int pos = 0; pos < hp.t2; ++pos) tab2freq[(size_t)kt1 * hp.t2 + pos] = kt1 + hp.t1 * order[pos];
    czt_tables(n, m, tab2freq, rp.chirp, rp.bhat);
    return 0;
}


// per-plane output/input table of the two-level column transform: for plane k1' the level-B transform
// P[k2] equals X[k1' + X1*k2]; by Hermitian symmetry X[(X1-k1') + X1*k2] = conj(P[X2-1-k2]).
struct Col2EntryHost { int pos, slot, flags, pad; };
inline void build_col2_entries(const FkHostPlan& hp, const std::vector<int>& k2slot /* size nx/2+1, -1 = pruned */,
                               std::vector<int>& plane_ptr, std::vector<Col2EntryHost>& ents) {
    const int nx = hp.nx, x1 = hp.x1, x2 = hp.x2;
    plane_ptr.assign((size_t)hp.planes + 1, 0);
    ents.clear();
    auto slot_of = [&](int k) { return (k >= 0 && 2 * k <= nx) ? k2slot[k] : -1; };
    for (int pl = 0; pl < hp.planes; ++pl) {
        plane_ptr[pl] = (int)ents.size();
        const bool self = (pl == 0) || (2 * pl == x1);
        for (int k2 = 0; k2 < x2; ++k2) {
            const int k = pl + x1 * k2;
            if (2 * k <= nx) {                               // direct: P[k2] = X[k]
                const int sl = slot_of(k);
                if (sl >= 0) ents.push_back({hp.pos_x2[k2], sl, 2, 0});
            } else {                                         // upper half: P[k2] = conj(X[nx - k]) (inverse only)
                const int sl = slot_of(nx - k);
                if (sl >= 0 && self) ents.push_back({hp.pos_x2[k2], sl, 1, 0});
            }
        }
        if (!self) {
            for (int k2 = 0; k2 < x2; ++k2) {                // mirror plane: X[(x1-pl) + x1*k2] = conj(P[x2-1-k2])
                const int kk = (x1 - pl) + x1 * k2;
                const int sl = slot_of(kk);
                if (sl >= 0) ents.push_back({hp.pos_x2[x2 - 1 - k2], sl, 3, 0});
            }
            // entries of this plane above nx/2 whose mirror lies in the partner plane are exactly the ones above
        }
    }
    plane_ptr[hp.planes] = (int)ents.size();
}

// dense per-plane table for the fused level-B kernels: need[plane][k2] = (direct slot, mirror slot code)
inline void build_col2_need(const FkHostPlan& hp, const std::vector<int>& k2slot, std::vector<int2>& need) {
    const int nx = hp.nx, x1 = hp.x1, x2 = hp.x2;
    need.assign((size_t)hp.planes * x2, make_int2(-1, -1));
    auto slot_of = [&](int k) { return (k >= 0 && 2 * k <= nx) ? k2slot[k] : -1; };
    for (int pl = 0; pl < hp.planes; ++pl) {
        const bool self = (pl == 0) || (2 * pl == x1);
        for (int k2 = 0; k2 < x2; ++k2) {
            int2& e = need[(size_t)pl * x2 + k2];
            const int k = pl + x1 * k2;
            if (2 * k <= nx) e.x = slot_of(k);
            else if (self) { const int sl = slot_of(nx - k); if (sl >= 0) e.y = -2 - sl; }      // inverse only
        }
        if (!self)
            for (int k2 = 0; k2 < x2; ++k2) {
                const int sl = slot_of((x1 - pl) + x1 * k2);
                if (sl >= 0) need[(size_t)pl * x2 + (x2 - 1 - k2)].y = sl;
            }
    }
}

}  // namespace d4w
