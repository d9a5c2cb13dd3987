// fft_plan.hpp -- host-side planning for the shared-memory FFT engine: radix schedule,
// twiddle table (double -> fp32, rounded once) and digit-reversal maps.
#pragma once
#include <cmath>
#include <map>
#include <string>
#include <vector>
#include <algorithm>
#include "fft_smem.cuh"

namespace d4w {

inline const std::vector<int>& inreg_radices() {
    static const std::vector<int> r = {25, 20, 16, 15, 12, 10, 8, 6, 5, 4, 3, 2};
    return r;
}

// Stage order used everywhere: generic primes first, then even radices (descending), then odd ones, so the
// late short-stride stages have odd strides.
inline std::vector<int> order_radices(const std::vector<int>& generic, const std::vector<int>& smooth) {
    std::vector<int> ev, od;
    for (int r : smooth) (r % 2 == 0 ? ev : od).push_back(r);
    std::sort(ev.rbegin(), ev.rend());
    std::sort(od.rbegin(), od.rend());
    std::vector<int> order = generic;
    order.insert(order.end(), ev.begin(), ev.end());
    order.insert(order.end(), od.begin(), od.end());
    return order;
}

// Cost model of one plan (scripts/bank_conflict_sim.py in C++): sum over stages of
//   butterfly rounds = ceil((n/r)/threads)  x  shared-memory wavefronts per ideal wavefront,
// where `lanes` = 8 for the 16-byte dual elements (quarter-warp phases), 16 for 8-byte elements.
inline double plan_cost(int n, const std::vector<int>& order, int threads, int lanes) {
    double total = 0.0;
    int ns = n;
    for (int r : order) {
        const int L = ns / r, per = n / r;
        long wf = 0, cnt = 0;
        const int step = std::max(1, per / 512) * lanes;          // sample the lane groups of long stages
        for (int id0 = 0; id0 < per; id0 += step) {
            int groups[16];
            for (int q = 0; q < r; ++q) {
                for (int g = 0; g < lanes; ++g) groups[g] = 0;
                int mx = 0;
                for (int i = id0; i < std::min(per, id0 + lanes); ++i) {
                    const int b = i / L, nn = i - b * L;
                    const int g = (int)(((long)b * ns + nn + (long)q * L) % lanes);
                    mx = std::max(mx, ++groups[g]);
                }
                wf += mx; ++cnt;
            }
        }
        const double conflict = cnt ? (double)wf / (double)cnt : 1.0;
        const double rounds = (double)((per + threads - 1) / threads);
        total += rounds * conflict;
        ns = L;
    }
    return total;
}

// minimum-stage split of a 2^a 3^b 5^c number into in-register radices <= max_radix; among the splits
// with the fewest stages pick the cheapest under plan_cost (DESIGN.md section 4).
inline bool split_smooth(int m, int max_radix, std::vector<int>& out, int n_total = 0, int threads = 256, int lanes = 16,
                         const std::vector<int>& generic = std::vector<int>()) {
    if (n_total <= 0) n_total = m;
    std::vector<int> best, cur;
    double best_cost = -1.0;
    size_t best_size = 0;
    struct Rec {
        int maxr, n_total, threads, lanes; const std::vector<int>& generic;
        std::vector<int>& best; double& best_cost; size_t& best_size; std::vector<int>& cur;
        void go(int m, int last) {
            if (m == 1) {
                if (!best.empty() && cur.size() > best_size) return;
                const double c = plan_cost(n_total, order_radices(generic, cur), threads, lanes);
                if (best.empty() || cur.size() < best_size || c < best_cost) { best = cur; best_cost = c; best_size = cur.size(); }
                return;
            }
            if (!best.empty() && cur.size() >= best_size) return;
            for (int r : inreg_radices()) {
                if (r > maxr || r > last || m % r) continue;
                cur.push_back(r);
                go(m / r, r);
                cur.pop_back();
            }
        }
    } rec{max_radix, n_total, threads, lanes, generic, best, best_cost, best_size, cur};
    rec.go(m, 1 << 30);
    out = best;
    return m == 1 || !best.empty();
}

// Build the stage schedule for length n.  Primes 7..61 become generic stages (first, where
// the leg spacing is long and contiguous); then even radices (descending), then odd ones, so
// the late short-stride stages are odd strides (bank-conflict free for 8-byte words).
inline bool make_plan(int n, int max_radix, FftPlan& pl, std::string& err, int threads = 256, int lanes = 16) {
    if (n < 1) { err = "FFT length must be >= 1"; return false; }
    std::vector<int> generic;
    int m = n;
    for (int p = 7; p <= 61 && m > 1; p += 2) {
        bool prime = true;
        for (int d = 3; d * d <= p; d += 2) if (p % d == 0) prime = false;
        if (!prime) continue;
        while (m % p == 0) { generic.push_back(p); m /= p; }
    }
    int t = m;
    while (t % 2 == 0) t /= 2;
    while (t % 3 == 0) t /= 3;
    while (t % 5 == 0) t /= 5;
    if (t != 1) {
        err = "unsupported FFT length " + std::to_string(n) + ": prime factor > 61";
        return false;
    }
    std::vector<int> smooth;
    if (m > 1 && !split_smooth(m, max_radix, smooth, n, threads, lanes, generic)) { err = "cannot factor " + std::to_string(n); return false; }
    std::vector<int> order = order_radices(generic, smooth);
    if ((int)order.size() > kMaxStages) { err = "too many FFT stages"; return false; }
    pl.n = n;
    pl.nstages = (int)order.size();
    int len = n;
    for (int s = 0; s < kMaxStages; ++s) { pl.radix[s] = 1; pl.sub[s] = 1; }
    for (int s = 0; s < pl.nstages; ++s) { pl.radix[s] = order[s]; pl.sub[s] = len; len /= order[s]; }
    return true;
}

// explicit stage order "20,20,25" (tuning knob); returns false if it does not multiply to n
inline bool make_plan_from_string(int n, const char* spec, FftPlan& pl) {
    std::vector<int> order;
    long long prod = 1;
    for (const char* c = spec; *c;) {
        int v = 0;
        while (*c >= '0' && *c <= '9') { v = v * 10 + (*c - '0'); ++c; }
        if (v < 2) return false;
        order.push_back(v); prod *= v;
        if (*c == ',' || *c == 'x') ++c; else if (*c) return false;
    }
    if (prod != n || (int)order.size() > kMaxStages) return false;
    pl.n = n; pl.nstages = (int)order.size();
    int len = n;
    for (int s = 0; s < kMaxStages; ++s) { pl.radix[s] = 1; pl.sub[s] = 1; }
    for (int s = 0; s < pl.nstages; ++s) { pl.radix[s] = order[s]; pl.sub[s] = len; len /= order[s]; }
    return true;
}

inline std::vector<float2> make_twiddles(int n) {
    std::vector<float2> t((size_t)std::max(n, 1));
    const double two_pi = 6.283185307179586476925286766559;
    for (int j = 0; j < n; ++j) {
        // exact octant reduction keeps the table symmetric and accurate to 0.5 ulp
        double a = two_pi * (double)j / (double)n;
        t[j] = make_float2((float)std::cos(a), (float)(-std::sin(a)));
    }
    return t;
}

inline std::vector<int> make_pos2freq(const FftPlan& pl) {
    std::vector<int> v(pl.n);
    for (int p = 0; p < pl.n; ++p) v[p] = pos_to_freq(pl, p);
    return v;
}

// true when n has a prime factor above 61, i.e. make_plan cannot build a mixed-radix schedule for it
inline bool has_prime_factor_above_61(int n) {
    for (int p = 2; p <= 61 && n > 1; ++p)
        while (n % p == 0) n /= p;
    return n > 1;
}

// smallest 2^a 3^b 5^c >= n
inline int next_5smooth(int n) {
    for (int m = std::max(n, 1);; ++m) {
        int t = m;
        while (t % 2 == 0) t /= 2;
        while (t % 3 == 0) t /= 3;
        while (t % 5 == 0) t /= 5;
        if (t == 1) return m;
    }
}

// forward DFT (exp(-2 pi i jk / n)) in double of a 2^a 3^b 5^c length, recursive decimation in time; host-side
// table building only (the chirp-z kernel spectrum)
inline void dft_5smooth_double(std::vector<double>& re, std::vector<double>& im) {
    const int n = (int)re.size();
    if (n <= 1) return;
    const int r = (n % 2 == 0) ? 2 : (n % 3 == 0) ? 3 : 5;
    const int m = n / r;
    std::vector<std::vector<double>> sre(r, std::vector<double>(m)), sim(r, std::vector<double>(m));
    for (int q = 0; q < r; ++q)
        for (int j = 0; j < m; ++j) { sre[q][j] = re[(size_t)j * r + q]; sim[q][j] = im[(size_t)j * r + q]; }
    for (int q = 0; q < r; ++q) dft_5smooth_double(sre[q], sim[q]);
    const double two_pi = 6.283185307179586476925286766559;
    for (int k = 0; k < n; ++k) {
        double ar = 0.0, ai = 0.0;
        for (int q = 0; q < r; ++q) {
            const long long e = (long long)q * k % n;                 // exact reduction of the twiddle exponent
            const double a = -two_pi * (double)e / (double)n, c = std::cos(a), s = std::sin(a);
            const double xr = sre[q][k % m], xi = sim[q][k % m];
            ar += xr * c - xi * s;
            ai += xr * s + xi * c;
        }
        re[k] = ar; im[k] = ai;
    }
}

}  // namespace d4w
