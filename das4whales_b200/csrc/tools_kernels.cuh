// tools_kernels.cuh -- __host__ __device__ bodies of the Gaussian-blurred f-k fan (tools.fk_filt_chunk, tools.py:27-49, and
// the legacy dsp.fk_filt, dsp.py:883-953) and of the per-row moments / linear detrend (scipy.signal.detrend(type='linear'),
// tools._energy_TimeDomain_chunk).  The same bodies run on the GPU (d4w_tools.cu) and on the host (tests/host_emul).
//
// The fan before the blur, G = g + fliplr(g) - g2 - fliplr(g2) with g = [f < k c_min and f < -k c_min], is a sum of four
// signed index intervals along every row: f_j = (j - ns/2) fval increases with j, so [f_j < k c and f_j < -k c] holds on a
// prefix [0, J) of the row, and its np.fliplr on the suffix [ns - J, ns).  The axis-1 blur of G is therefore exact from the
// cumulative Gaussian weights (no input read), and only the axis-0 blur needs the 2r + 1 taps.  scipy.ndimage blurs axis 0
// first; the two passes commute, so only the rounding of the float64 sums differs.
#pragma once
#include <cmath>
#include <cstring>

namespace d4w {

constexpr int kFanTJ = 32;                      // columns per CTA (one per lane)
constexpr int kFanU = 8;                        // consecutive output rows per thread
constexpr int kFanG = 8;                        // row groups (warps) per CTA
constexpr int kFanRT = kFanU * kFanG;           // output rows per CTA
constexpr int kFanThreads = kFanTJ * kFanG;

// scipy.ndimage.gaussian_filter's default truncate = 4: radius = int(4 sigma + 0.5)
__host__ __device__ inline int fan_radius(double sigma) { return (int)(4.0 * sigma + 0.5); }
// taps read by the sliding accumulation: 2r + U rounded up to U (the weights beyond 2r are zero)
__host__ __device__ inline int fan_steps(int r) { return (2 * r + kFanU + kFanU - 1) / kFanU * kFanU; }
__host__ __device__ inline int fan_tile_rows(int r) { return kFanRT + 2 * r + kFanU; }
__host__ __device__ inline size_t fan_smem_bytes(int r) {
    return sizeof(double) * ((size_t)fan_steps(r) + (size_t)(2 * r + 2) + (size_t)fan_tile_rows(r) * kFanTJ);
}
// workspace: min / max keys, weights w[2r + 1], cumulative weights cw[2r + 2], the row prefixes J[nx][2]
__host__ __device__ inline size_t fan_ws_bytes(int nx, int r) {
    return 16 + sizeof(double) * ((size_t)(2 * r + 1) + (size_t)(2 * r + 2)) + sizeof(int) * 2 * (size_t)nx;
}

struct FanParams {
    int nx, ns, r;
    double kval, fval, c_min, c_max;
    const double* w;    // [2r + 1]
    const double* cw;   // [2r + 2], cw[m] = w[0] + ... + w[m - 1]
    const int* J;       // [nx][2]
};

// scipy.ndimage 'reflect' (d c b a | a b c d | d c b a), repeated for any p: the extension has period 2n
__host__ __device__ inline int reflect_index(long long p, int n) {
    const long long two = 2LL * n;
    long long m = p % two;
    if (m < 0) m += two;
    return (int)(m < n ? m : two - 1 - m);
}

// number of columns j with f_j < prod and f_j < -prod, f_j = (j - ns/2) * fval as numpy.fft.fftfreq forms it; fval > 0 makes
// the set a prefix, found by bisection on the reference's own comparisons
__host__ __device__ inline int fan_prefix(int ns, double fval, double prod) {
    int lo = 0, hi = ns;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const double f = (double)(mid - ns / 2) * fval;
        if (f < prod && f < -prod) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// row i: k_i = (i - nx/2) * kval; J[i] = the prefixes of g (c_min) and g2 (c_max), products in the reference's order (kk * c)
__host__ __device__ inline void body_fan_row(int nx, int ns, double kval, double fval, double c_min, double c_max, int* J, int i) {
    const double k = (double)(i - nx / 2) * kval;
    J[2 * i] = fan_prefix(ns, fval, k * c_min);
    J[2 * i + 1] = fan_prefix(ns, fval, k * c_max);
}

// scipy.ndimage._gaussian_kernel1d(sigma, 0, r): exp(-0.5 / sigma^2 * x^2), x = -r..r, over its sum; and the running sums
__host__ __device__ inline void fan_weights(double sigma, int r, double* w, double* cw) {
    const double c = -0.5 / (sigma * sigma);
    double s = 0.0;
    for (int x = -r; x <= r; ++x) {
        w[x + r] = exp(c * (double)((long long)x * x));
        s += w[x + r];
    }
    cw[0] = 0.0;
    for (int m = 0; m <= 2 * r; ++m) {
        w[m] /= s;
        cw[m + 1] = cw[m] + w[m];
    }
}

__host__ __device__ inline long long floor_div(long long a, long long b) {
    const long long q = a / b;
    return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

// sum_{s = -r..r} w_s [reflect(j + s) in [a, b)]: every copy of [a, b) in the period-2n extension that meets the window
// [j - r, j + r] adds a difference of cumulative weights
__host__ __device__ inline double interval_blur(const double* cw, int r, int n, int a, int b, int j) {
    if (a >= b) return 0.0;
    const long long lo = (long long)j - r, hi = (long long)j + r + 1, two = 2LL * n;
    double acc = 0.0;
    for (long long q = floor_div(lo, two) - 1; q <= floor_div(hi - 1, two); ++q) {
        const long long base = q * two;
        const long long c0[2] = {base + a, base + two - b}, c1[2] = {base + b, base + two - a};
        for (int h = 0; h < 2; ++h) {
            const long long s = c0[h] > lo ? c0[h] : lo, e = c1[h] < hi ? c1[h] : hi;
            if (s < e) acc += cw[e - j + r] - cw[s - j + r];
        }
    }
    return acc;
}

// the axis-1 blur of G at row i (already reflected into [0, nx)), column j.  [0, J1) - [0, J2) is the signed interval between
// the two prefixes (likewise the suffixes), so a row where g = g2 blurs to exactly 0, as scipy's does
__host__ __device__ inline double fan_row_blur(const FanParams& p, const double* cw, int i, int j) {
    const int j1 = p.J[2 * i], j2 = p.J[2 * i + 1], n = p.ns;
    const int lo = j1 < j2 ? j1 : j2, hi = j1 < j2 ? j2 : j1;
    const double v = interval_blur(cw, p.r, n, lo, hi, j) + interval_blur(cw, p.r, n, n - hi, n - lo, j);
    return j1 < j2 ? -v : v;
}

__host__ __device__ inline double row_blur(const FanParams& p, const double* cw, int i, int j) { return fan_row_blur(p, cw, i, j); }

// The tile and tap bodies below serve every mask whose rows are index intervals before the blur: P supplies nx, ns, r, the
// weights w / cw and row_blur(p, cw, i, j), the exact axis-1 blur of row i (FanParams here, DesignParams further down).
// shared copies of the weights, zero-padded to wz[fan_steps(r)], and of cw[2r + 2]
template <class P>
__host__ __device__ inline void body_fan_weights(const P& p, double* wz, double* cw, int tid, int nthr) {
    const int S = fan_steps(p.r);
    for (int s = tid; s < S; s += nthr) wz[s] = s <= 2 * p.r ? p.w[s] : 0.0;
    for (int m = tid; m < 2 * p.r + 2; m += nthr) cw[m] = p.cw[m];
}
// CTA (i0, j0): the shared tile H[tr][c] = axis-1 blur at row reflect(i0 - r + tr), column j0 + c
template <class P>
__host__ __device__ inline void body_fan_fill_tile(const P& p, int i0, int j0, const double* cw, double* H, int tid, int nthr) {
    const int rows = fan_tile_rows(p.r);
    for (int idx = tid; idx < rows * kFanTJ; idx += nthr) {
        const int tr = idx / kFanTJ, c = idx % kFanTJ, j = j0 + c;
        H[idx] = j < p.ns ? row_blur(p, cw, reflect_index((long long)i0 - p.r + tr, p.nx), j) : 0.0;
    }
}

// thread (g, lane): acc[u] = sum_{t = 0..2r} w[t] H[g U + u + t][lane], the axis-0 blur at row i0 + g U + u.  Each tile value
// is read once and feeds U accumulators; the U weights in flight sit in a register ring (static indices after unrolling).
template <class P>
__host__ __device__ inline void body_fan_taps(const P& p, const double* wz, const double* H, int g, int lane, double* acc) {
    double wr[kFanU];
#pragma unroll
    for (int u = 0; u < kFanU; ++u) { acc[u] = 0.0; wr[u] = 0.0; }
    const int S = fan_steps(p.r);
    const double* col = H + (size_t)g * kFanU * kFanTJ + lane;
    for (int s0 = 0; s0 < S; s0 += kFanU) {
#pragma unroll
        for (int v = 0; v < kFanU; ++v) {
            const double d = col[(size_t)(s0 + v) * kFanTJ];
            wr[v] = wz[s0 + v];
#pragma unroll
            for (int u = 0; u < kFanU; ++u) acc[u] = fma(wr[(v - u + kFanU) % kFanU], d, acc[u]);
        }
    }
}

// order-preserving map of a double onto unsigned 64-bit keys (for atomicMin / atomicMax); NaN is never produced here
__host__ __device__ inline unsigned long long fan_key(double x) {
    unsigned long long b;
    memcpy(&b, &x, 8);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__host__ __device__ inline double fan_unkey(unsigned long long k) {
    const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    double x;
    memcpy(&x, &b, 8);
    return x;
}

// ---- the hybrid, hybrid_gs and hybrid_ninf_gs masks of dsp.py:174-305, :457-579, :582-702 ---------------------------------
// Shifted layout: f_j = (j - ns/2) fval, k_i = (i - nx/2) kval as numpy.fft.fftfreq forms them.  col_lo / col_hi are the
// reference's np.argmax column range (the loop over [col_lo, col_hi) does not run when col_hi <= col_lo).
//
// hybrid: elementwise, A[i, j] = H_j c(i, j) inside [col_lo, col_hi) and H_j outside, then A[i, j] + A[i, ns-1-j] (fliplr).
// hybrid_gs: before the sigma = 20 blur, row i of M + fliplr(M) is 1 on S_i and on its mirror, S_i = {H_j = 1} ∩ ({j in
// [col_lo, col_hi) : -kp_j < k_i < kp_j} ∪ {j outside [col_lo, col_hi)}), kp_j = f_j / cp_min.  kp_j does not decrease with j
// (cp_min > 0), so both comparisons first fail and then hold: S_i is the H band cut to [0, col_lo) ∪ [s_i, ns).
// hybrid_ninf_gs: the blur commutes with fliplr and flipud (a symmetric kernel, 'reflect' mode), so blur(M) + its fliplr, then
// + its flipud, is the blur of the sum of rows i and nx-1-i of M and their mirrors.  Inside [col_lo, col_hi) M is 1 where
// k_i > -(f_j / cp_min), a suffix, and k_i < -(f_j / cp_max), a prefix: S_i = H ∩ ([0, col_lo) ∪ [s_i, e_i) ∪ [col_hi, ns)).
// Each row is a short list of index intervals (overlaps count twice, as the sums do), blurred along axis 1 by interval_blur
// and along axis 0 by the fan's tile and taps.
constexpr int kDesignHybrid = 0, kDesignHybridGs = 1, kDesignHybridNinfGs = 2;
constexpr double kDesignSigma = 20.0;              // ndimage.gaussian_filter(M, 20), dsp.py:540 and :659
constexpr int kDesignMaxIv = 12;                   // 3 pieces x fliplr x flipud
constexpr int kDesignStride = 1 + 2 * kDesignMaxIv;  // per row: count, then [a, b) pairs

struct DesignParams {
    int kind, nx, ns, r;
    double kval, fval, cs_min, cp_min, cp_max;
    int col_lo, col_hi, h_lo, h_hi;     // [h_lo, h_hi): where H_j = 1 (gs kinds)
    const double* H;                    // [ns] (hybrid)
    const double* w;                    // [2r + 1]
    const double* cw;                   // [2r + 2]
    int* iv;                            // [nx][kDesignStride]
};

// workspace: w[2r + 1], cw[2r + 2], H[ns], then the row intervals
__host__ __device__ inline size_t design_ws_bytes(int nx, int ns, int r) {
    return sizeof(double) * ((size_t)(4 * r + 3) + (size_t)ns) + sizeof(int) * (size_t)kDesignStride * (size_t)nx;
}

// [h_lo, h_hi) = the columns where a gs mask's H is 1; false unless H is 1 on that one band and 0 elsewhere
__host__ __device__ inline bool design_h_band(const double* H, int ns, int* h_lo, int* h_hi) {
    int j = 0;
    while (j < ns && H[j] == 0.0) ++j;
    *h_lo = j;
    while (j < ns && H[j] == 1.0) ++j;
    *h_hi = j;
    while (j < ns && H[j] == 0.0) ++j;
    return j == ns;
}

// the reference's column factor of the hybrid mask (dsp.py:246-262): the -sin ramp, then the sin ramp (both only when
// ks != kp), then the passband's 1
__host__ __device__ inline double hybrid_col(double k, double f, double cs_min, double cp_min) {
    const double ks = f / cs_min, kp = f / cp_min;
    double c = 0.0;
    if (ks != kp) {
        if (k >= -ks && k <= -kp) c = -sin(0.5 * M_PI * (k + ks) / (kp - ks));
        if (-k >= -ks && -k <= -kp) c = sin(0.5 * M_PI * (k - ks) / (kp - ks));
    }
    if (k < kp && k > -kp) c = 1.0;
    return c;
}

__host__ __device__ inline double hybrid_half(const DesignParams& p, double k, int j) {
    const double v = p.H[j];
    return j >= p.col_lo && j < p.col_hi ? v * hybrid_col(k, (double)(j - p.ns / 2) * p.fval, p.cs_min, p.cp_min) : v;
}

__host__ __device__ inline double body_hybrid(const DesignParams& p, int i, int j) {
    const double k = (double)(i - p.nx / 2) * p.kval;
    return hybrid_half(p, k, j) + hybrid_half(p, k, p.ns - 1 - j);
}

// which = 0: -kp < k < kp (hybrid_gs); 1: k > -(f / cp_min); 2: not k < -(f / cp_max).  Each first fails, then holds, as j grows.
__host__ __device__ inline bool design_pred(int which, double k, double f, double cp_min, double cp_max) {
    if (which == 0) {
        const double kp = f / cp_min;
        return k < kp && k > -kp;
    }
    if (which == 1) return k > -(f / cp_min);
    return !(k < -(f / cp_max));
}

// first j in [lo, hi) where design_pred holds (hi when it never does), by bisection on the reference's comparisons
__host__ __device__ inline int design_first(int which, int lo, int hi, int ns, double fval, double k, double cp_min, double cp_max) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (design_pred(which, k, (double)(mid - ns / 2) * fval, cp_min, cp_max)) hi = mid; else lo = mid + 1;
    }
    return lo;
}

// append [a, b) ∩ H and its fliplr mirror to a row's list
__host__ __device__ inline void design_push(const DesignParams& p, int* row, int a, int b) {
    a = a > p.h_lo ? a : p.h_lo;
    b = b < p.h_hi ? b : p.h_hi;
    if (a >= b) return;
    const int n = row[0];
    row[1 + 2 * n] = a; row[2 + 2 * n] = b;
    row[3 + 2 * n] = p.ns - b; row[4 + 2 * n] = p.ns - a;
    row[0] = n + 2;
}

// S_m (row m of M before the blur) and its mirror, appended to row
__host__ __device__ inline void design_row_set(const DesignParams& p, int m, int* row) {
    const double k = (double)(m - p.nx / 2) * p.kval;
    const int lo = p.col_lo, hi = p.col_hi > lo ? p.col_hi : lo;
    design_push(p, row, 0, lo);
    if (p.kind == kDesignHybridGs) {
        design_push(p, row, design_first(0, lo, hi, p.ns, p.fval, k, p.cp_min, p.cp_max), p.ns);
    } else {
        design_push(p, row, design_first(1, lo, hi, p.ns, p.fval, k, p.cp_min, p.cp_max),
                    design_first(2, lo, hi, p.ns, p.fval, k, p.cp_min, p.cp_max));
        design_push(p, row, hi, p.ns);
    }
}

// row i's interval list: S_i for hybrid_gs; S_i and S_{nx-1-i} for hybrid_ninf_gs (the flipud partner; itself at an odd nx's
// centre row, which the sum counts twice)
__host__ __device__ inline void body_design_row(const DesignParams& p, int i) {
    int* row = p.iv + (size_t)i * kDesignStride;
    row[0] = 0;
    design_row_set(p, i, row);
    if (p.kind == kDesignHybridNinfGs) design_row_set(p, p.nx - 1 - i, row);
}

__host__ __device__ inline double row_blur(const DesignParams& p, const double* cw, int i, int j) {
    const int* row = p.iv + (size_t)i * kDesignStride;
    double v = 0.0;
    for (int q = 0; q < row[0]; ++q) v += interval_blur(cw, p.r, p.ns, row[1 + 2 * q], row[2 + 2 * q], j);
    return v;
}

// ---- per-row moments over time chunks, and the linear detrend --------------------------------------------------------------
// partial sums of one thread over the chunk [c0, c0 + len) of a row: s[0] = sum x, s[1] = sum t x (t from 0 at the chunk
// start), s[2] = sum x^2, in float64
__host__ __device__ inline void body_moments(const float* row, int len, int tid, int nthr, double* s) {
    double a = 0.0, b = 0.0, q = 0.0;
    for (int t = tid; t < len; t += nthr) {
        const double v = row[t];
        a += v;
        b = fma((double)t, v, b);
        q = fma(v, v, q);
    }
    s[0] = a; s[1] = b; s[2] = q;
}

// y = x - (least-squares line of the n samples): mean + slope (t - (n - 1)/2), slope = sum (t - (n-1)/2) x / (n (n^2 - 1) / 12)
__host__ __device__ inline float detrend_sample(float x, int t, int n, const double* m) {
    const double mean = m[0] / n, h = 0.5 * (n - 1);
    const double den = (double)n * ((double)n * n - 1.0) / 12.0;
    const double slope = n > 1 ? (m[1] - h * m[0]) / den : 0.0;
    return (float)((double)x - mean - slope * ((double)t - h));
}

}  // namespace d4w
