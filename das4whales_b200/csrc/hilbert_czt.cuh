// hilbert_czt.cuh -- analytic signal of rows whose length n has no mixed-radix split (chirp-z / Bluestein rows), and the
// epilogues every Hilbert route shares.
//
// With c[t] = exp(-i pi (t^2 mod 2n) / n), a convolution length m >= 2n - 1 and bhat = FFT_m(conj c, wrapped) / m
// (fk_hostplan.hpp: czt_tables), the analytic signal with scipy.signal.hilbert's weights h (h/n, or sgn/n when two real rows
// share one complex transform) is
//   1. u = x c for t < n, 0 for n <= t < m
//   2. v = IFFT_m(FFT_m(u) bhat)                      -> X[f] = c[f] v[f]
//   3. z[f] = (h[f]/n) v[f] for f < n, 0 for f >= n     (the chirps between the two DFTs cancel)
//   4. w = IFFT_m(FFT_m(z) conj bhat)                 (c is even, so the second kernel's spectrum is conj bhat)
//   5. a[t] = conj(c[t]) w[t] for t < n, then hilbert_epilogue / hilbert_epilogue2.
// Whole-row route (m <= 16 384): one CTA runs the four m-point transforms in shared memory (body_hczt_row).  Split route
// (m = T1 x T2): body_hczt_fwd -> k_row_mid(_fused)_c with bhat -> body_hczt_turn (inverse T1 split, step 3 and forward T1
// split in registers: for a given t2 both splits touch the index set {t2 + j T2}) -> k_row_mid(_fused)_c with conj bhat ->
// body_hczt_inv.  Bodies are __host__ __device__ functions of (block, tid, nthr, smem) so tests/host_emul runs them too.
#pragma once
#include "fk_kernels.cuh"

namespace d4w {

// EPI_HILB: the Hilbert transform H(x) itself (dsp.instant_freq needs the phase); EPI_ENVSTD: envelope / std_row
// (improcess.trace2image, improcess.py:61)
enum { EPI_ENV = 0, EPI_SNR = 1, EPI_HILB = 2, EPI_ENVSTD = 3 };

__host__ __device__ __forceinline__ float hilbert_epilogue(float2 z, int mode, float var) {
    if (mode == EPI_HILB) return z.y;
    const float p = z.x * z.x + z.y * z.y;
    if (mode == EPI_ENVSTD) return sqrtf(p) / sqrtf(var);
    return mode == EPI_ENV ? sqrtf(p) : 10.0f * log10f(p / var);
}

// two real rows per complex transform: x is the row itself, h its Hilbert transform (see k_hsplit_inv2)
__host__ __device__ __forceinline__ float hilbert_epilogue2(float x, float h, int mode, float var) {
    if (mode == EPI_HILB) return h;
    const float p = x * x + h * h;
    if (mode == EPI_ENVSTD) return sqrtf(p) / sqrtf(var);
    return mode == EPI_ENV ? sqrtf(p) : 10.0f * log10f(p / var);
}

struct HcztParams {
    int n, m, t2;                 // row length, convolution length, m / T1
    int nx;                       // rows in this call
    int pair;                     // two real rows per complex transform (weights sgn/n)
    float invn;                   // 1 / n
    const float2* chirp;          // c[t], t < n
    const float2* twT;            // W_m^j, j < t2 (split twiddles)
};

// scipy.signal.hilbert's weight at frequency f < n, over n: 1 at DC (and Nyquist), 2 below n/2, 0 above; minus 1 for pairs
__host__ __device__ __forceinline__ float hczt_weight(const HcztParams& hp, int f) {
    float w = (f == 0 || 2 * f == hp.n) ? 1.f : (2 * f < hp.n ? 2.f : 0.f);
    if (hp.pair) w -= 1.f;
    return w * hp.invn;
}

// ---- whole row in one CTA (T1 == 1): smem holds the m-point row
__host__ __device__ inline void body_hczt_row(const RowParams& rp, const HcztParams& hp, const float2* __restrict__ bhat,
                                              const float2* __restrict__ bhatc, const float* __restrict__ x, float* __restrict__ out,
                                              int mode, const double* __restrict__ stats, int row, int tid, int nthr, float2* smem) {
    const int n = hp.n, m = hp.m, nst = rp.pl.nstages;
    const float* src = x + (size_t)row * n;
    for (int i = tid; i < m; i += nthr) smem[i] = (i < n) ? cscale(hp.chirp[i], src[i]) : make_float2(0.f, 0.f);
    D4W_SYNC();
    fft_forward_stages(smem, rp.pl, rp.tw, 1, m, tid, nthr, 0, nst);
    for (int i = tid; i < m; i += nthr) smem[i] = cmul(smem[i], bhat[i]);
    D4W_SYNC();
    fft_inverse_stages(smem, rp.pl, rp.tw, 1, m, tid, nthr, 0, nst);
    for (int i = tid; i < m; i += nthr) smem[i] = (i < n) ? cscale(smem[i], hczt_weight(hp, i)) : make_float2(0.f, 0.f);
    D4W_SYNC();
    fft_forward_stages(smem, rp.pl, rp.tw, 1, m, tid, nthr, 0, nst);
    for (int i = tid; i < m; i += nthr) smem[i] = cmul(smem[i], bhatc[i]);
    D4W_SYNC();
    fft_inverse_stages(smem, rp.pl, rp.tw, 1, m, tid, nthr, 0, nst);
    const float var = (mode == EPI_SNR || mode == EPI_ENVSTD) ? (float)stats[4 * (size_t)row + 2] : 1.f;
    float* dst = out + (size_t)row * n;
    for (int i = tid; i < n; i += nthr) dst[i] = hilbert_epilogue(cmulc(smem[i], hp.chirp[i]), mode, var);
}

// ---- split route, step 1: forward radix-T1 split of u = x c (zero from n on); workspace row pr holds rows 2pr, 2pr+1 as
// a + i b when hp.pair, else row pr
template <int T1>
__host__ __device__ inline void body_hczt_fwd(const HcztParams& hp, const float* __restrict__ x, float2* __restrict__ w, int pr, int t2) {
    const int n = hp.n, t2len = hp.t2;
    const int ra = hp.pair ? 2 * pr : pr;
    const bool has_b = hp.pair && ra + 1 < hp.nx;
    const float* sa = x + (size_t)ra * n;
    float2 v[T1];
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        const int t = t2 + j * t2len;
        v[j] = (t < n) ? cmul(make_float2(sa[t], has_b ? sa[(size_t)n + t] : 0.f), hp.chirp[t]) : make_float2(0.f, 0.f);
    });
    float2 p[T1];
    twiddle_powers<T1>(hp.twT[t2], p);
    DFT<T1, false>::run(v);
    float2* dst = w + (size_t)pr * hp.m + t2;
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; dst[(size_t)j * t2len] = (j > 0) ? cmul(v[j], p[j]) : v[j]; });
}

// ---- step 3: inverse split of the first convolution, weights (natural frequency order, zero from n on), forward split of
// the second -- all on the T1 values of one t2 in registers
template <int T1>
__host__ __device__ inline void body_hczt_turn(const HcztParams& hp, float2* __restrict__ w, int pr, int t2) {
    const int t2len = hp.t2;
    float2* base = w + (size_t)pr * hp.m + t2;
    float2 v[T1];
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; v[j] = base[(size_t)j * t2len]; });
    float2 p[T1];
    twiddle_powers<T1>(hp.twT[t2], p);
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j > 0) v[j] = cmulc(v[j], p[j]); });
    DFT<T1, true>::run(v);
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        const int f = t2 + j * t2len;
        v[j] = (f < hp.n) ? cscale(v[j], hczt_weight(hp, f)) : make_float2(0.f, 0.f);
    });
    DFT<T1, false>::run(v);
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; base[(size_t)j * t2len] = (j > 0) ? cmul(v[j], p[j]) : v[j]; });
}

// ---- step 5: inverse split, times conj(c[t]), epilogue.  Pairs: with s = IFFT(sgn (A + i B)) = i H(a) - H(b),
// H(a) = Im s and H(b) = -Re s
template <int T1>
__host__ __device__ inline void body_hczt_inv(const HcztParams& hp, const float2* __restrict__ w, const float* __restrict__ x,
                                              float* __restrict__ out, int mode, const double* __restrict__ stats, int pr, int t2) {
    const int n = hp.n, t2len = hp.t2;
    const float2* src = w + (size_t)pr * hp.m + t2;
    float2 v[T1];
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; v[j] = src[(size_t)j * t2len]; });
    float2 p[T1];
    twiddle_powers<T1>(hp.twT[t2], p);
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j > 0) v[j] = cmulc(v[j], p[j]); });
    DFT<T1, true>::run(v);
    const size_t ra = hp.pair ? 2 * (size_t)pr : (size_t)pr;
    const bool has_b = hp.pair && ra + 1 < (size_t)hp.nx;
    const bool need_var = mode == EPI_SNR || mode == EPI_ENVSTD;
    const float va = need_var ? (float)stats[4 * ra + 2] : 1.f;
    const float vb = (need_var && has_b) ? (float)stats[4 * (ra + 1) + 2] : 1.f;
    const float* xa = x + ra * n;
    float* oa = out + ra * n;
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        const int t = t2 + j * t2len;
        if (t < n) {
            const float2 z = cmulc(v[j], hp.chirp[t]);
            if (!hp.pair) {
                oa[t] = hilbert_epilogue(z, mode, va);
            } else {
                oa[t] = hilbert_epilogue2(xa[t], z.y, mode, va);
                if (has_b) oa[(size_t)n + t] = hilbert_epilogue2(xa[(size_t)n + t], -z.x, mode, vb);
            }
        }
    });
}

#ifdef __CUDACC__
// the direct rows' middle passes with a complex table (B^ or conj B^)
static __global__ void __launch_bounds__(256, 2)
k_row_mid_c(RowParams rp, float2* __restrict__ w, size_t ldw, const float2* __restrict__ tab, size_t tab_slot_stride) {
    body_row_mid(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(256, 2)
k_row_mid_fused_c(RowParams rp, float2* __restrict__ w, size_t ldw, const float2* __restrict__ tab, size_t tab_slot_stride) {
    body_row_mid_fused(rp, w, ldw, tab, tab_slot_stride, blockIdx.x, blockIdx.y, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

static __global__ void __launch_bounds__(256, 2)
k_hczt_row(RowParams rp, HcztParams hp, const float2* __restrict__ bhat, const float2* __restrict__ bhatc, const float* __restrict__ x,
           float* __restrict__ out, int mode, const double* __restrict__ stats) {
    body_hczt_row(rp, hp, bhat, bhatc, x, out, mode, stats, blockIdx.x, threadIdx.x, blockDim.x, d4w_dyn_smem);
}

template <int T1>
static __global__ void __launch_bounds__(128)
k_hczt_fwd(HcztParams hp, const float* __restrict__ x, float2* __restrict__ w) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 < hp.t2) body_hczt_fwd<T1>(hp, x, w, blockIdx.y, t2);
}

template <int T1>
static __global__ void __launch_bounds__(128)
k_hczt_turn(HcztParams hp, float2* __restrict__ w) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 < hp.t2) body_hczt_turn<T1>(hp, w, blockIdx.y, t2);
}

template <int T1>
static __global__ void __launch_bounds__(128)
k_hczt_inv(HcztParams hp, const float2* __restrict__ w, const float* __restrict__ x, float* __restrict__ out, int mode,
           const double* __restrict__ stats) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 < hp.t2) body_hczt_inv<T1>(hp, w, x, out, mode, stats, blockIdx.y, t2);
}
#endif  // __CUDACC__

}  // namespace d4w
