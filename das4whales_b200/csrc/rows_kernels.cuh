// rows_kernels.cuh -- per-channel (row) operators: statistics, overlap-save matched filter,
// Hilbert envelope / SNR, forward-backward SOS IIR, batched STFT magnitude.
//
// Reference arithmetic replaced (files under /root/reference/src/das4whales/):
//   detect.compute_cross_correlogram / shift_xcorr          detect.py:96-166
//   dsp.snr_tr_array, |scipy.signal.hilbert| (pick_times_env) dsp.py:956-976, detect.py:192
//   dsp.bp_filt (scipy filtfilt) and caller-side sosfiltfilt dsp.py:859-880, Example.py:55
//   dsp.get_spectrogram / detect.get_sliced_nspectrogram     dsp.py:41-78, detect.py:334-408
#pragma once
#include <cuda_fp16.h>
#include "fft_pfa.cuh"
#include <type_traits>
#include "fft_smem.cuh"
#include "fk_kernels.cuh"
#include "hilbert_czt.cuh"

namespace d4w {

// ------------------------------------------------------------------ row statistics
// stats[row] = {mean, absmax, population variance, 0}; optional segpre[row][s] = sum over
// samples before segment s of (x - mean)/absmax  (prefix of the normalised row, for the
// matched filter's mean-of-padded-template term, SURVEY App. A.3).
constexpr int kMaxSeg = 512;

static __global__ void __launch_bounds__(256)
k_row_stats(const float* __restrict__ x, int ns, int seglen, int nseg, double* __restrict__ stats,
            double* __restrict__ segpre) {
    __shared__ double s_sum[8], s_sq[8];
    __shared__ float s_max[8];
    __shared__ double s_seg[kMaxSeg];
    const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const float* r = x + (size_t)row * ns;
    double sum = 0.0, sq = 0.0;
    float mx = 0.f;
    if (segpre) for (int s = tid; s < nseg; s += blockDim.x) s_seg[s] = 0.0;
    __syncthreads();
    if (segpre) {
        // one warp per segment keeps the per-segment sums exact and atomic-free
        for (int s = wid; s < nseg; s += 8) {
            const int a = s * seglen, b = min(ns, a + seglen);
            double ss = 0.0;
            int i = a + lane;
            // four independent loads in flight per lane (the accumulation chain must not serialise the memory latency)
            for (; i + 96 < b; i += 128) {
                const float v0 = r[i], v1 = r[i + 32], v2 = r[i + 64], v3 = r[i + 96];
                ss += ((double)v0 + (double)v1) + ((double)v2 + (double)v3);
                sq += ((double)v0 * (double)v0 + (double)v1 * (double)v1) + ((double)v2 * (double)v2 + (double)v3 * (double)v3);
                mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v0), fabsf(v1))), fmaxf(fabsf(v2), fabsf(v3)));
            }
            for (; i < b; i += 32) {
                const float v = r[i];
                ss += (double)v; sq += (double)v * (double)v; mx = fmaxf(mx, fabsf(v));
            }
            for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
            if (lane == 0) s_seg[s] = ss;
            sum += ss / 32.0;     // every lane adds 1/32 of the warp total -> warp reduction below restores it
        }
    } else {
        int i = tid;
        const int st = blockDim.x;
        for (; i + 3 * st < ns; i += 4 * st) {
            const float v0 = r[i], v1 = r[i + st], v2 = r[i + 2 * st], v3 = r[i + 3 * st];
            sum += ((double)v0 + (double)v1) + ((double)v2 + (double)v3);
            sq += ((double)v0 * (double)v0 + (double)v1 * (double)v1) + ((double)v2 * (double)v2 + (double)v3 * (double)v3);
            mx = fmaxf(fmaxf(mx, fmaxf(fabsf(v0), fabsf(v1))), fmaxf(fabsf(v2), fabsf(v3)));
        }
        for (; i < ns; i += st) {
            const float v = r[i];
            sum += (double)v; sq += (double)v * (double)v; mx = fmaxf(mx, fabsf(v));
        }
    }
    for (int o = 16; o > 0; o >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, o);
        sq += __shfl_xor_sync(0xffffffffu, sq, o);
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (lane == 0) { s_sum[wid] = sum; s_sq[wid] = sq; s_max[wid] = mx; }
    __syncthreads();
    if (tid == 0) {
        double S = 0.0, Q = 0.0; float M = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { S += s_sum[w]; Q += s_sq[w]; M = fmaxf(M, s_max[w]); }
        const double mean = S / ns;
        double var = Q / ns - mean * mean;
        if (var < 0.0) var = 0.0;
        stats[4 * (size_t)row + 0] = mean;
        stats[4 * (size_t)row + 1] = (double)M;
        stats[4 * (size_t)row + 2] = var;
        stats[4 * (size_t)row + 3] = 0.0;
        if (segpre) {
            double acc = 0.0;
            for (int s = 0; s < nseg; ++s) {
                segpre[(size_t)row * nseg + s] = acc;
                const int len = min(ns, (s + 1) * seglen) - s * seglen;
                acc += (s_seg[s] - mean * len) / (double)M;
            }
        }
    }
}

// ------------------------------------------------------------------ SNR (no envelope)
static __global__ void k_snr_plain(const float* __restrict__ x, float* __restrict__ out, int ns, const double* __restrict__ stats,
                            size_t total) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t row = i / ns;
    const float var = (float)stats[4 * row + 2];
    const float v = x[i];
    out[i] = 10.0f * log10f(v * v / var);                 // dsp.py:976 (zeros give -inf like the reference)
}

// ------------------------------------------------------------------ overlap-save matched filter
// One block = two consecutive segments of one channel packed as re/im of one complex FFT of
// length nb (correlation with a real template is real-linear, so no untangling is needed):
//   S = FFT(seg);  for each template: IFFT(S * conj(C_t)/nb/m_t) -> valid = nb - L + 1 lags.
// tabs[t][p] holds conj(C_t[k(p)]) / (nb * m_t) in transform order.
struct XcorrParams {
    FftPlan pl;
    const float2* tw;
    int nb, valid, ntpl, ns, normalize, nseg;
};

// SAME = true: the centred ("same") correlation of scripts/main_gabordetect.py:245, scipy.signal.correlate(x / max(x), c,
// 'same'), for templates whose taps are prepended with zeros up to a common lag offset lag0 (d4w_xcorr_same).  The block
// that produces outputs t .. t + V - 1 reads samples t - lag0 .., zero outside [0, ns), scaled by 1 / rowmax[row]; there is
// no demeaning and no mu term, and a row whose maximum is not > 0 is all zeros (its CTAs write zeros and return before any
// transform: the branch is uniform, row = blockIdx.y).  SAME = false ignores rowmax and lag0.
// sample t of a row in SAME mode (t may be negative)
__device__ __forceinline__ float xcorr_same_load(const float* __restrict__ r, int t, int ns, float inv) {
    return (t >= 0 && t < ns) ? r[t] * inv : 0.f;
}
// zeros for output samples [a, b) of one row, every template
__device__ __forceinline__ void xcorr_zero_span(float* __restrict__ out, size_t out_tpl_stride, int ntpl, size_t row_off, int a, int b,
                                                int tid, int nthr) {
    for (int t = 0; t < ntpl; ++t) {
        float* o = out + (size_t)t * out_tpl_stride + row_off;
        for (int i = a + tid; i < b; i += nthr) o[i] = 0.f;
    }
}

template <bool SAME>
static __global__ void __launch_bounds__(128, 4)
k_xcorr(XcorrParams xp, const float* __restrict__ x, const float2* __restrict__ tabs, const double* __restrict__ stats,
        const double* __restrict__ segpre, const double* __restrict__ mu_over_m, float* __restrict__ out, size_t out_tpl_stride,
        const float* __restrict__ rowmax, int lag0) {
    extern __shared__ float2 sm[];
    float2* S = sm;                   // spectrum of the segment pair
    float2* B = sm + xp.nb;           // work buffer for the inverse
    float2* P = sm + 2 * xp.nb;       // exclusive prefix sums of the normalised samples (valid entries)
    __shared__ float2 s_wsum[32];
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, wid = tid >> 5;
    const int row = blockIdx.y;
    const int seg_a = 2 * blockIdx.x, seg_b = seg_a + 1;
    const int ns = xp.ns, nb = xp.nb, V = xp.valid;
    const int ta = seg_a * V, tb = seg_b * V;
    const float* r = x + (size_t)row * ns;
    float mean = 0.f, inv = 1.f;
    if constexpr (SAME) {
        const float m = rowmax[row];
        if (!(m > 0.f)) { xcorr_zero_span(out, out_tpl_stride, xp.ntpl, (size_t)row * ns, ta, min(ns, ta + 2 * V), tid, nthr); return; }
        inv = 1.f / m;
    } else {
        if (xp.normalize) { mean = (float)stats[4 * (size_t)row]; inv = (float)(1.0 / stats[4 * (size_t)row + 1]); }
    }
    for (int i = tid; i < nb; i += nthr) {
        const int ia = ta + i, ib = tb + i;
        if constexpr (SAME) {
            S[i] = make_float2(xcorr_same_load(r, ia - lag0, ns, inv), xcorr_same_load(r, ib - lag0, ns, inv));
        } else {
            const float a = (ia < ns) ? (r[ia] - mean) * inv : 0.f;
            const float b = (ib < ns) ? (r[ib] - mean) * inv : 0.f;
            S[i] = make_float2(a, b);
        }
    }
    __syncthreads();
    // exclusive prefix of the first V samples of each segment (only needed for the mu term)
    if (!SAME && xp.normalize) {
        const int chunk = (V + nthr - 1) / nthr;
        const int i0 = min(V, tid * chunk), i1 = min(V, i0 + chunk);
        float2 loc = make_float2(0.f, 0.f);
        for (int i = i0; i < i1; ++i) { loc.x += S[i].x; loc.y += S[i].y; }
        float2 inc = loc;
        for (int o = 1; o < 32; o <<= 1) {
            const float ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
            if (lane >= o) { inc.x += ux; inc.y += uy; }
        }
        if (lane == 31) s_wsum[wid] = inc;
        __syncthreads();
        float2 base = make_float2(0.f, 0.f);
        for (int w = 0; w < wid; ++w) { base.x += s_wsum[w].x; base.y += s_wsum[w].y; }
        float2 run = make_float2(base.x + inc.x - loc.x, base.y + inc.y - loc.y);
        const float pa = (seg_a < xp.nseg) ? (float)segpre[(size_t)row * xp.nseg + seg_a] : 0.f;
        const float pb = (seg_b < xp.nseg) ? (float)segpre[(size_t)row * xp.nseg + seg_b] : 0.f;
        for (int i = i0; i < i1; ++i) {
            P[i] = make_float2(pa + run.x, pb + run.y);
            run.x += S[i].x; run.y += S[i].y;
        }
        __syncthreads();
    }
    fft_forward_stages(S, xp.pl, xp.tw, 1, nb, tid, nthr, 0, xp.pl.nstages);
    for (int t = 0; t < xp.ntpl; ++t) {
        const float2* tab = tabs + (size_t)t * nb;
        for (int i = tid; i < nb; i += nthr) B[i] = cmul(S[i], tab[i]);
        __syncthreads();
        fft_inverse_stages(B, xp.pl, xp.tw, 1, nb, tid, nthr, 0, xp.pl.nstages);
        const float mu = (!SAME && xp.normalize) ? (float)mu_over_m[t] : 0.f;
        float* o = out + (size_t)t * out_tpl_stride + (size_t)row * ns;
        for (int i = tid; i < V; i += nthr) {
            const float2 v = B[i];
            float2 p = make_float2(0.f, 0.f);
            if (!SAME && xp.normalize) p = P[i];
            // out = (sum x~ c - mu * suffix) / m, suffix = -prefix because x~ sums to zero
            if (ta + i < ns) o[ta + i] = v.x + mu * p.x;
            if (tb + i < ns) o[tb + i] = v.y + mu * p.y;
        }
        __syncthreads();
    }
}

// ---- fused variant (plans with >= 2 stages whose first and last stage are in-register radices) -------------------
// Passes over shared memory per block: load + prefix, forward stages 0 .. n-2, then per template ONE pass doing the last
// forward stage, the multiply with the template spectrum and the first inverse stage in registers (S is left intact for
// the next template), the middle inverse stages, and the last inverse stage straight to global memory with the mu term.
// Table order: tabs[t][m * (nb / RL) + j] belongs to engine position j * RL + m (d4w_fft_plan_table_order).
template <int R>
__device__ __forceinline__ void xcorr_last_fused(const float2* __restrict__ S, float2* __restrict__ B, const float2* __restrict__ tab,
                                                 int nb, int tid, int nthr) {
    const int G = nb / R;
    for (int j = tid; j < G; j += nthr) {
        float2 v[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = S[j * R + q]; });
        DFT<R, false>::run(v);
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = cmul(v[m], tab[m * G + j]); });
        DFT<R, true>::run(v);
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; B[j * R + q] = v[q]; });
    }
}
template <int R>
__device__ __forceinline__ void xcorr_first_inv_out(const float2* __restrict__ B, const float2* __restrict__ P, const float2* __restrict__ tw,
                                                    int nb, int V, int ta, int tb, int ns, float mu, bool use_p, float* __restrict__ o,
                                                    int tid, int nthr) {
    const int L = nb / R;
    for (int n = tid; n < L; n += nthr) {
        float2 v[R], p[R];
        twiddle_powers<R>(tw[n], p);
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; const float2 u = B[n + m * L]; v[m] = (m > 0) ? cmulc(u, p[m]) : u; });
        DFT<R, true>::run(v);
        static_for<R>([&](auto qc) {
            constexpr int q = decltype(qc)::value;
            const int i = n + q * L;
            if (i < V) {
                float2 pr = make_float2(0.f, 0.f);
                if (use_p) pr = P[i];
                if (ta + i < ns) o[ta + i] = v[q].x + mu * pr.x;
                if (tb + i < ns) o[tb + i] = v[q].y + mu * pr.y;
            }
        });
    }
}

template <bool SAME>
static __global__ void __launch_bounds__(128, 4)
k_xcorr_fused(XcorrParams xp, const float* __restrict__ x, const float2* __restrict__ tabs, const double* __restrict__ stats,
              const double* __restrict__ segpre, const double* __restrict__ mu_over_m, float* __restrict__ out, size_t out_tpl_stride,
              const float* __restrict__ rowmax, int lag0) {
    extern __shared__ float2 sm[];
    float2* S = sm;
    float2* B = sm + xp.nb;
    float2* P = sm + 2 * xp.nb;
    __shared__ float2 s_wsum[32];
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, wid = tid >> 5;
    const int row = blockIdx.y;
    const int seg_a = 2 * blockIdx.x, seg_b = seg_a + 1;
    const int ns = xp.ns, nb = xp.nb, V = xp.valid, nst = xp.pl.nstages;
    const int ta = seg_a * V, tb = seg_b * V;
    const float* r = x + (size_t)row * ns;
    float mean = 0.f, inv = 1.f;
    if constexpr (SAME) {
        const float m = rowmax[row];
        if (!(m > 0.f)) { xcorr_zero_span(out, out_tpl_stride, xp.ntpl, (size_t)row * ns, ta, min(ns, ta + 2 * V), tid, nthr); return; }
        inv = 1.f / m;
    } else {
        if (xp.normalize) { mean = (float)stats[4 * (size_t)row]; inv = (float)(1.0 / stats[4 * (size_t)row + 1]); }
    }
    for (int i = tid; i < nb; i += nthr) {
        const int ia = ta + i, ib = tb + i;
        if constexpr (SAME) {
            S[i] = make_float2(xcorr_same_load(r, ia - lag0, ns, inv), xcorr_same_load(r, ib - lag0, ns, inv));
        } else {
            const float a = (ia < ns) ? (r[ia] - mean) * inv : 0.f;
            const float b = (ib < ns) ? (r[ib] - mean) * inv : 0.f;
            S[i] = make_float2(a, b);
        }
    }
    __syncthreads();
    if (!SAME && xp.normalize) {
        const int chunk = (V + nthr - 1) / nthr;
        const int i0 = min(V, tid * chunk), i1 = min(V, i0 + chunk);
        float2 loc = make_float2(0.f, 0.f);
        for (int i = i0; i < i1; ++i) { loc.x += S[i].x; loc.y += S[i].y; }
        float2 inc = loc;
        for (int o = 1; o < 32; o <<= 1) {
            const float ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
            if (lane >= o) { inc.x += ux; inc.y += uy; }
        }
        if (lane == 31) s_wsum[wid] = inc;
        __syncthreads();
        float2 base = make_float2(0.f, 0.f);
        for (int w = 0; w < wid; ++w) { base.x += s_wsum[w].x; base.y += s_wsum[w].y; }
        float2 run = make_float2(base.x + inc.x - loc.x, base.y + inc.y - loc.y);
        const float pa = (seg_a < xp.nseg) ? (float)segpre[(size_t)row * xp.nseg + seg_a] : 0.f;
        const float pb = (seg_b < xp.nseg) ? (float)segpre[(size_t)row * xp.nseg + seg_b] : 0.f;
        for (int i = i0; i < i1; ++i) {
            P[i] = make_float2(pa + run.x, pb + run.y);
            run.x += S[i].x; run.y += S[i].y;
        }
        __syncthreads();
    }
    fft_forward_stages(S, xp.pl, xp.tw, 1, nb, tid, nthr, 0, nst - 1);
    const int r0 = xp.pl.radix[0], rl = xp.pl.radix[nst - 1];
    for (int t = 0; t < xp.ntpl; ++t) {
        const float2* tab = tabs + (size_t)t * nb;
#define D4W_CALL(R) xcorr_last_fused<R>(S, B, tab, nb, tid, nthr);
        D4W_ROW_RADIX_SWITCH(rl, D4W_CALL)
#undef D4W_CALL
        __syncthreads();
        fft_inverse_stages(B, xp.pl, xp.tw, 1, nb, tid, nthr, 1, nst - 1);
        const float mu = (!SAME && xp.normalize) ? (float)mu_over_m[t] : 0.f;
        float* o = out + (size_t)t * out_tpl_stride + (size_t)row * ns;
#define D4W_CALL(R) xcorr_first_inv_out<R>(B, P, xp.tw, nb, V, ta, tb, ns, mu, !SAME && xp.normalize != 0, o, tid, nthr);
        D4W_ROW_RADIX_SWITCH(r0, D4W_CALL)
#undef D4W_CALL
        __syncthreads();
    }
}

// ---- dual-lane variant: FOUR consecutive segments of one channel per CTA as the two f32x2 lanes of the dual engine ---------
// Element i of the block is the 16-byte cpd {x = (seg_a[i], seg_c[i]), y = (seg_b[i], seg_d[i])}: lane A is the complex
// signal a + i b, lane B is c + i d, and both lanes run through one instruction stream of butterflies whose twiddles are
// formed once for the two lanes (each lane operation is a scalar FFMA / FADD / FMUL, fft_dual.cuh).
// The template spectra are lane-independent scalars (dmul_s).  Shared memory: S and B as cpd (16 B x nb each) and the
// exclusive prefix sums of the mu term as a float4 per 8 samples; the output sweep adds the <= 7 samples before each output
// in its group, re-read from the input in fp32 (an fp16 per-sample remainder in shared memory cost up to 3e-5 l2 error
// when mu / m is large: short rows, templates with a large mean).

template <int R>
__device__ __forceinline__ void xcorrd_last_fused(const cpd* __restrict__ S, cpd* __restrict__ B, const float2* __restrict__ tab,
                                                  int nb, int tid, int nthr) {
    const int G = nb / R;
    for (int j = tid; j < G; j += nthr) {
        cpd v[R], u[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = S[j * R + q]; });
        DFTD<R, false>::run(v);                                                  // X[m] at v[outpos(m)]
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; u[m] = dmul_s(v[outpos<R>(m)], tab[m * G + j]); });
        DFTD<R, true>::run(u);
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; B[j * R + q] = u[outpos<R>(q)]; });
    }
}
template <int R>
__device__ __forceinline__ void xcorrd_first_inv_out(const cpd* __restrict__ B, const float4* __restrict__ Pc, const float* __restrict__ r,
                                                     float mean, float inv, const float2* __restrict__ tw, int nb, int V, int t0, int ns,
                                                     float mu, bool use_p, float* __restrict__ o, int tid, int nthr) {
    const int L = nb / R;
    for (int n = tid; n < L; n += nthr) {
        cpd v[R];
        static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; v[m] = B[n + m * L]; });
        if (L > 1) apply_stage_twiddles<R, true, false>(v, tw[n]);
        DFTD<R, true>::run(v);
        static_for<R>([&](auto qc) {
            constexpr int q = decltype(qc)::value;
            const int i = n + q * L;
            if (i < V) {
                const cpd z = v[outpos<R>(q)];
                float va = f2x_lo(z.x), vc = f2x_hi(z.x), vb = f2x_lo(z.y), vd = f2x_hi(z.y);
                const int ta = t0 + i, tb = ta + V, tc = tb + V, td = tc + V;
                if (use_p) {
                    // exclusive prefix = group prefix + the <= 7 normalised samples before i in its group, re-read in fp32
                    float4 c = Pc[i >> 3];
                    for (int k = i & ~7; k < i; ++k) {
                        const int ka = t0 + k, kb = ka + V, kc = kb + V, kd = kc + V;
                        c.x += (ka < ns) ? (r[ka] - mean) * inv : 0.f;
                        c.y += (kb < ns) ? (r[kb] - mean) * inv : 0.f;
                        c.z += (kc < ns) ? (r[kc] - mean) * inv : 0.f;
                        c.w += (kd < ns) ? (r[kd] - mean) * inv : 0.f;
                    }
                    va += mu * c.x; vb += mu * c.y; vc += mu * c.z; vd += mu * c.w;
                }
                if (ta < ns) o[ta] = va;
                if (tb < ns) o[tb] = vb;
                if (tc < ns) o[tc] = vc;
                if (td < ns) o[td] = vd;
            }
        });
    }
}

// Small-radix dispatch: the dual kernel is compiled for radices <= 10 only, so that its register allocation (the maximum
// over every path in the kernel) stays <= 128 and two 256-thread CTAs share an SM (16 warps); blocks are planned as
// 10 . 10 . 5 . 5 (2500) etc.: 250 - 500 butterflies per stage keep all 256 threads busy.
#define D4W_SMALL_RADIX_SWITCH(r, CALL)                                                                       \
    switch (r) {                                                                                              \
        case 2: { CALL(2) } break; case 3: { CALL(3) } break; case 4: { CALL(4) } break; case 5: { CALL(5) } break;         \
        case 6: { CALL(6) } break; case 8: { CALL(8) } break; default: { CALL(10) } break;                                   \
    }
__host__ __device__ inline bool xcorr_dual_radix_ok(int r) { return r == 2 || r == 3 || r == 4 || r == 5 || r == 6 || r == 8 || r == 10; }
template <bool INV>
__device__ __forceinline__ void stage_dispatch_dual_small(cpd* s, const float2* tw, int n_total, int ns, int r, int tid, int nthr) {
#define D4W_CALL(R) stage_dual<R, INV>(s, tw, n_total, ns, 1, n_total, tid, nthr);
    D4W_SMALL_RADIX_SWITCH(r, D4W_CALL)
#undef D4W_CALL
}

template <bool SAME>
static __global__ void __launch_bounds__(256, 2)
k_xcorr_dual(XcorrParams xp, const float* __restrict__ x, const float2* __restrict__ tabs, const double* __restrict__ stats,
             const double* __restrict__ segpre, const double* __restrict__ mu_over_m, float* __restrict__ out, size_t out_tpl_stride,
             const float* __restrict__ rowmax, int lag0) {
    extern __shared__ __align__(16) unsigned char smraw[];
    const int ns = xp.ns, nb = xp.nb, V = xp.valid, nst = xp.pl.nstages;
    const int ng = (V + 7) >> 3;                           // prefix groups of 8 samples
    cpd* S = reinterpret_cast<cpd*>(smraw);
    cpd* B = S + nb;
    float4* Pc = reinterpret_cast<float4*>(B + nb);
    __shared__ float4 s_wsum[8];
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31, wid = tid >> 5;
    const int row = blockIdx.y;
    const int seg0 = 4 * blockIdx.x;
    const int t0 = seg0 * V;
    const float* r = x + (size_t)row * ns;
    float mean = 0.f, inv = 1.f;
    if constexpr (SAME) {
        const float m = rowmax[row];
        if (!(m > 0.f)) { xcorr_zero_span(out, out_tpl_stride, xp.ntpl, (size_t)row * ns, t0, min(ns, t0 + 4 * V), tid, nthr); return; }
        inv = 1.f / m;
    } else {
        if (xp.normalize) { mean = (float)stats[4 * (size_t)row]; inv = (float)(1.0 / stats[4 * (size_t)row + 1]); }
    }
    for (int i = tid; i < nb; i += nthr) {
        const int ia = t0 + i, ib = ia + V, ic = ib + V, id = ic + V;
        if constexpr (SAME) {
            const float a = xcorr_same_load(r, ia - lag0, ns, inv), b = xcorr_same_load(r, ib - lag0, ns, inv);
            const float c = xcorr_same_load(r, ic - lag0, ns, inv), d = xcorr_same_load(r, id - lag0, ns, inv);
            S[i] = dmake(f2x_set(a, c), f2x_set(b, d));
        } else {
            const float a = (ia < ns) ? (r[ia] - mean) * inv : 0.f;
            const float b = (ib < ns) ? (r[ib] - mean) * inv : 0.f;
            const float c = (ic < ns) ? (r[ic] - mean) * inv : 0.f;
            const float d = (id < ns) ? (r[id] - mean) * inv : 0.f;
            S[i] = dmake(f2x_set(a, c), f2x_set(b, d));
        }
    }
    __syncthreads();
    if (!SAME && xp.normalize) {
        // exclusive prefix of the first V samples of each of the four segments: thread -> contiguous run of groups
        const int gpt = (ng + nthr - 1) / nthr;
        const int g0 = min(ng, tid * gpt), g1 = min(ng, g0 + gpt);
        float4 loc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = g0 * 8; i < min(V, g1 * 8); ++i) {
            const cpd z = S[i];
            loc.x += f2x_lo(z.x); loc.y += f2x_lo(z.y); loc.z += f2x_hi(z.x); loc.w += f2x_hi(z.y);
        }
        float4 inc = loc;
        for (int o = 1; o < 32; o <<= 1) {
            const float ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
            const float uz = __shfl_up_sync(0xffffffffu, inc.z, o), uw = __shfl_up_sync(0xffffffffu, inc.w, o);
            if (lane >= o) { inc.x += ux; inc.y += uy; inc.z += uz; inc.w += uw; }
        }
        if (lane == 31) s_wsum[wid] = inc;
        __syncthreads();
        float4 run = make_float4(inc.x - loc.x, inc.y - loc.y, inc.z - loc.z, inc.w - loc.w);
        for (int w = 0; w < wid; ++w) { run.x += s_wsum[w].x; run.y += s_wsum[w].y; run.z += s_wsum[w].z; run.w += s_wsum[w].w; }
        const size_t sp = (size_t)row * xp.nseg + seg0;
        run.x += (seg0 + 0 < xp.nseg) ? (float)segpre[sp + 0] : 0.f;
        run.y += (seg0 + 1 < xp.nseg) ? (float)segpre[sp + 1] : 0.f;
        run.z += (seg0 + 2 < xp.nseg) ? (float)segpre[sp + 2] : 0.f;
        run.w += (seg0 + 3 < xp.nseg) ? (float)segpre[sp + 3] : 0.f;
        for (int g = g0; g < g1; ++g) {
            Pc[g] = run;
            float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int i = g * 8; i < min(V, g * 8 + 8); ++i) {
                const cpd z = S[i];
                f.x += f2x_lo(z.x); f.y += f2x_lo(z.y); f.z += f2x_hi(z.x); f.w += f2x_hi(z.y);
            }
            run.x += f.x; run.y += f.y; run.z += f.z; run.w += f.w;
        }
        __syncthreads();
    }
    for (int st = 0; st < nst - 1; ++st) {
        stage_dispatch_dual_small<false>(S, xp.tw, nb, xp.pl.sub[st], xp.pl.radix[st], tid, nthr);
        __syncthreads();
    }
    const int r0 = xp.pl.radix[0], rl = xp.pl.radix[nst - 1];
    for (int t = 0; t < xp.ntpl; ++t) {
        const float2* tab = tabs + (size_t)t * nb;
#define D4W_CALL(R) xcorrd_last_fused<R>(S, B, tab, nb, tid, nthr);
        D4W_SMALL_RADIX_SWITCH(rl, D4W_CALL)
#undef D4W_CALL
        __syncthreads();
        for (int st = nst - 2; st >= 1; --st) {
            stage_dispatch_dual_small<true>(B, xp.tw, nb, xp.pl.sub[st], xp.pl.radix[st], tid, nthr);
            __syncthreads();
        }
        const float mu = (!SAME && xp.normalize) ? (float)mu_over_m[t] : 0.f;
        float* o = out + (size_t)t * out_tpl_stride + (size_t)row * ns;
#define D4W_CALL(R) xcorrd_first_inv_out<R>(B, Pc, r, mean, inv, xp.tw, nb, V, t0, ns, mu, !SAME && xp.normalize != 0, o, tid, nthr);
        D4W_SMALL_RADIX_SWITCH(r0, D4W_CALL)
#undef D4W_CALL
        __syncthreads();
    }
}

// ---- prime-factor variant (blocks of 2520 = 5 * 7 * 8 * 9 samples, fft_pfa.cuh): same four-segments-per-CTA dual-lane layout,
// but no twiddle factors between the stages and conflict-free strides.  The block is loaded in natural time order (B),
// prefix-summed, scattered to the 4-D positions (S), transformed, and the result is gathered back to time order on the way out
// so that every global access stays coalesced.  tabs[t][m * 280 + j] belongs to position j * 9 + m (d4w_fft_plan_table_order).
// Exclusive prefix of the mu term in k_xcorr_pfa: a float4 per group of 8 samples (Pc) plus the in-group remainder per sample
// in fp16 (Pf; an fp32 remainder would not fit two CTAs per SM).  The remainder is a sum of <= 7 normalised samples,
// |.| <= 14, so its fp16 rounding is <= 7e-3 and costs <= 1e-7 on the output while |mu / m| <= 2^-16 -- the script's chirps
// on rows of >= 1 500 samples.  Larger |mu / m| (templates with a visible mean, short rows) would see it (up to 3e-5 l2 with
// a 300-tap Hann pulse on 400-sample rows): the output sweep then rebuilds the remainder in fp32 from the input instead.
struct __align__(8) half4 { __half2 ac, bd; };
constexpr float kXcorrMuFp16Max = 1.0f / 65536;
constexpr int kPfaThreads = 256;      // measured: 256 threads 10.8 ms, 320 threads 11.2 ms (10 000 x 120 000, HF + LF)
template <bool SAME>
static __global__ void __launch_bounds__(kPfaThreads, 2)
k_xcorr_pfa(XcorrParams xp, const int* __restrict__ tpos, const float* __restrict__ x, const float2* __restrict__ tabs,
            const double* __restrict__ stats, const double* __restrict__ segpre, const double* __restrict__ mu_over_m,
            float* __restrict__ out, size_t out_tpl_stride, const float* __restrict__ rowmax, int lag0) {
    extern __shared__ __align__(16) unsigned char smraw[];
    constexpr int nb = kPfaN;
    const int ns = xp.ns, V = xp.valid;
    const int ng = (V + 7) >> 3;
    cpd* S = reinterpret_cast<cpd*>(smraw);
    cpd* B = S + nb;
    float4* Pc = reinterpret_cast<float4*>(B + nb);
    half4* Pf = reinterpret_cast<half4*>(Pc + ng);
    const int tid = threadIdx.x, nthr = blockDim.x, lane = tid & 31;
    const int row = blockIdx.y;
    const int seg0 = 4 * blockIdx.x;
    const int t0 = seg0 * V;
    const float* r = x + (size_t)row * ns;
    float mean = 0.f, inv = 1.f;
    if constexpr (SAME) {
        const float m = rowmax[row];
        if (!(m > 0.f)) { xcorr_zero_span(out, out_tpl_stride, xp.ntpl, (size_t)row * ns, t0, min(ns, t0 + 4 * V), tid, nthr); return; }
        inv = 1.f / m;
    } else {
        if (xp.normalize) { mean = (float)stats[4 * (size_t)row]; inv = (float)(1.0 / stats[4 * (size_t)row + 1]); }
    }
    // load + normalise in time order (B) and, in the same sweep, the prefix sums of the mu term: lanes 8k .. 8k+7 hold one
    // prefix group, so a 3-step segmented shuffle scan gives the in-group exclusive prefix (Pf, fp16) and the group total
    // (parked in Pc, turned into the exclusive prefix over groups below) -- no shared-memory traffic, no bank conflicts
    for (int i0 = 0; i0 < nb; i0 += nthr) {                      // every lane runs every iteration (full-mask shuffles below)
        const int i = i0 + tid;
        const bool in = i < nb;
        const int ia = t0 + i, ib = ia + V, ic = ib + V, id = ic + V;
        if constexpr (SAME) {
            if (in) B[i] = dmake(f2x_set(xcorr_same_load(r, ia - lag0, ns, inv), xcorr_same_load(r, ic - lag0, ns, inv)),
                                 f2x_set(xcorr_same_load(r, ib - lag0, ns, inv), xcorr_same_load(r, id - lag0, ns, inv)));
            continue;                                             // no mu term
        }
        const float a = (in && ia < ns) ? (r[ia] - mean) * inv : 0.f;
        const float b = (in && ib < ns) ? (r[ib] - mean) * inv : 0.f;
        const float c = (in && ic < ns) ? (r[ic] - mean) * inv : 0.f;
        const float d = (in && id < ns) ? (r[id] - mean) * inv : 0.f;
        if (in) B[i] = dmake(f2x_set(a, c), f2x_set(b, d));
        if (xp.normalize) {
            float4 inc = make_float4(a, b, c, d);
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) {
                const float ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
                const float uz = __shfl_up_sync(0xffffffffu, inc.z, o), uw = __shfl_up_sync(0xffffffffu, inc.w, o);
                if ((lane & 7) >= o) { inc.x += ux; inc.y += uy; inc.z += uz; inc.w += uw; }
            }
            if (i < V) { half4 h; h.ac = __floats2half2_rn(inc.x - a, inc.z - c); h.bd = __floats2half2_rn(inc.y - b, inc.w - d); Pf[i] = h; }
            if ((lane & 7) == 7 && in && (i >> 3) < ng) Pc[i >> 3] = inc;
        }
    }
    __syncthreads();
    if (!SAME && xp.normalize && tid < 32) {
        // exclusive scan of the group totals by one warp, seeded with the row prefix at the start of each segment
        const size_t sp = (size_t)row * xp.nseg + seg0;
        float4 carry;
        carry.x = (seg0 + 0 < xp.nseg) ? (float)segpre[sp + 0] : 0.f;
        carry.y = (seg0 + 1 < xp.nseg) ? (float)segpre[sp + 1] : 0.f;
        carry.z = (seg0 + 2 < xp.nseg) ? (float)segpre[sp + 2] : 0.f;
        carry.w = (seg0 + 3 < xp.nseg) ? (float)segpre[sp + 3] : 0.f;
        for (int g0 = 0; g0 < ng; g0 += 32) {
            const int g = g0 + lane;
            const float4 own = (g < ng) ? Pc[g] : make_float4(0.f, 0.f, 0.f, 0.f);
            float4 inc = own;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const float ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
                const float uz = __shfl_up_sync(0xffffffffu, inc.z, o), uw = __shfl_up_sync(0xffffffffu, inc.w, o);
                if (lane >= o) { inc.x += ux; inc.y += uy; inc.z += uz; inc.w += uw; }
            }
            if (g < ng) Pc[g] = make_float4(carry.x + inc.x - own.x, carry.y + inc.y - own.y, carry.z + inc.z - own.z, carry.w + inc.w - own.w);
            carry.x += __shfl_sync(0xffffffffu, inc.x, 31); carry.y += __shfl_sync(0xffffffffu, inc.y, 31);
            carry.z += __shfl_sync(0xffffffffu, inc.z, 31); carry.w += __shfl_sync(0xffffffffu, inc.w, 31);
        }
    }
    pfa_first_from_time(B, S, tid, nthr);                       // radix-5 stage straight from the time-ordered block
    __syncthreads();
    pfa_forward_23(S, tid, nthr);
    for (int t = 0; t < xp.ntpl; ++t) {
        pfa_last_fused(S, B, tabs + (size_t)t * nb, tid, nthr);
        __syncthreads();
        pfa_inverse_3(B, tid, nthr);
        const float mu = (!SAME && xp.normalize) ? (float)mu_over_m[t] : 0.f;
        float* o = out + (size_t)t * out_tpl_stride + (size_t)row * ns;
        if (!SAME && xp.normalize && fabsf(mu) > kXcorrMuFp16Max) {
            for (int i0 = 0; i0 < V; i0 += nthr) {               // every lane runs every iteration (full-mask shuffles below)
                // in-group exclusive prefix in fp32: the load sweep's segmented scan again, on the samples re-read from the
                // input (L2-resident)
                const int i = i0 + tid;
                const int ta = t0 + i, tb = ta + V, tc = tb + V, td = tc + V;
                const float a = (i < V && ta < ns) ? (r[ta] - mean) * inv : 0.f;
                const float b = (i < V && tb < ns) ? (r[tb] - mean) * inv : 0.f;
                const float c = (i < V && tc < ns) ? (r[tc] - mean) * inv : 0.f;
                const float d = (i < V && td < ns) ? (r[td] - mean) * inv : 0.f;
                float4 inc = make_float4(a, b, c, d);
#pragma unroll
                for (int s = 1; s < 8; s <<= 1) {
                    const float ux = __shfl_up_sync(0xffffffffu, inc.x, s), uy = __shfl_up_sync(0xffffffffu, inc.y, s);
                    const float uz = __shfl_up_sync(0xffffffffu, inc.z, s), uw = __shfl_up_sync(0xffffffffu, inc.w, s);
                    if ((lane & 7) >= s) { inc.x += ux; inc.y += uy; inc.z += uz; inc.w += uw; }
                }
                if (i >= V) continue;
                const float4 g = Pc[i >> 3];
                const cpd z = B[tpos[i]];
                const float va = f2x_lo(z.x) + mu * (g.x + inc.x - a), vb = f2x_lo(z.y) + mu * (g.y + inc.y - b);
                const float vc = f2x_hi(z.x) + mu * (g.z + inc.z - c), vd = f2x_hi(z.y) + mu * (g.w + inc.w - d);
                if (ta < ns) o[ta] = va;
                if (tb < ns) o[tb] = vb;
                if (tc < ns) o[tc] = vc;
                if (td < ns) o[td] = vd;
            }
        } else {
            for (int i = tid; i < V; i += nthr) {
                const cpd z = B[tpos[i]];
                float va = f2x_lo(z.x), vc = f2x_hi(z.x), vb = f2x_lo(z.y), vd = f2x_hi(z.y);
                if (!SAME && xp.normalize) {
                    const float4 c = Pc[i >> 3];
                    const half4 f = Pf[i];
                    const float2 fac = __half22float2(f.ac), fbd = __half22float2(f.bd);
                    va += mu * (c.x + fac.x); vb += mu * (c.y + fbd.x); vc += mu * (c.z + fac.y); vd += mu * (c.w + fbd.y);
                }
                const int ta = t0 + i, tb = ta + V, tc = tb + V, td = tc + V;
                if (ta < ns) o[ta] = va;
                if (tb < ns) o[tb] = vb;
                if (tc < ns) o[tc] = vc;
                if (td < ns) o[td] = vd;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ Hilbert envelope / SNR on the T1 x T2 row engine
// EPI_* modes and hilbert_epilogue / hilbert_epilogue2: hilbert_czt.cuh (shared with the chirp-z rows)

// ---- split rows: two real rows per complex transform ------------------------------------------------------------
// The Hilbert transform is linear and maps real rows to real rows, so for z = a + i b one complex FFT -> (-i sgn f) -> IFFT
// yields H(a) + i H(b): half the transforms and half the workspace traffic of the analytic-signal route.  The middle
// pass multiplies by the real table sgn(f)/ns (0 at DC and Nyquist, scipy.signal.hilbert's h - 1); the factor -i is
// applied here: with u = IFFT(Z sgn), H(a) = Im u and H(b) = -Re u; |hilbert(a)| = sqrt(a^2 + H(a)^2).
template <int T1>
static __global__ void __launch_bounds__(128)
k_hsplit_fwd2(const float* __restrict__ x, int nx, int ns, float2* __restrict__ w, int t2len, const float2* __restrict__ twT) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 >= t2len) return;
    const size_t pr = blockIdx.y;
    const float* sa = x + (2 * pr) * (size_t)ns + t2;
    const bool has_b = 2 * pr + 1 < (size_t)nx;
    const float* sb = sa + ns;
    float2 v[T1];
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        v[j] = make_float2(sa[(size_t)j * t2len], has_b ? sb[(size_t)j * t2len] : 0.f);
    });
    float2 p[T1];
    twiddle_powers<T1>(twT[t2], p);
    DFT<T1, false>::run(v);
    float2* dst = w + pr * ns + t2;
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        dst[(size_t)j * t2len] = (j > 0) ? cmul(v[j], p[j]) : v[j];
    });
}
template <int T1>
static __global__ void __launch_bounds__(128)
k_hsplit_inv2(const float2* __restrict__ w, const float* __restrict__ x, int nx, int ns, float* __restrict__ out, int t2len,
              const float2* __restrict__ twT, int mode, const double* __restrict__ stats) {
    const int t2 = blockIdx.x * blockDim.x + threadIdx.x;
    if (t2 >= t2len) return;
    const size_t pr = blockIdx.y;
    const float2* src = w + pr * ns + t2;
    float2 v[T1];
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; v[j] = src[(size_t)j * t2len]; });
    float2 p[T1];
    twiddle_powers<T1>(twT[t2], p);
    static_for<T1>([&](auto jc) { constexpr int j = decltype(jc)::value; if constexpr (j > 0) v[j] = cmulc(v[j], p[j]); });
    DFT<T1, true>::run(v);
    const size_t ra = 2 * pr, rb = 2 * pr + 1;
    const bool has_b = rb < (size_t)nx;
    const bool need_var = mode == EPI_SNR || mode == EPI_ENVSTD;
    const float va = need_var ? (float)stats[4 * ra + 2] : 1.f;
    const float vb = (need_var && has_b) ? (float)stats[4 * rb + 2] : 1.f;
    const float* xa = x + ra * ns + t2;
    float* oa = out + ra * ns + t2;
    static_for<T1>([&](auto jc) {
        constexpr int j = decltype(jc)::value;
        const size_t o = (size_t)j * t2len;
        oa[o] = hilbert_epilogue2(xa[o], v[j].y, mode, va);
        if (has_b) oa[ns + o] = hilbert_epilogue2(xa[ns + o], -v[j].x, mode, vb);
    });
}

// whole row in one CTA (T1 == 1): real in -> FFT -> weights -> IFFT -> epilogue out
static __global__ void __launch_bounds__(256, 2)
k_hilbert_row(RowParams rp, const float* __restrict__ x, float* __restrict__ out, const float* __restrict__ tab, int mode,
              const double* __restrict__ stats) {
    extern __shared__ float2 sm[];
    const int n = rp.t2, tid = threadIdx.x, nthr = blockDim.x;
    const size_t row = blockIdx.x;
    const float* src = x + row * n;
    for (int i = tid; i < n; i += nthr) sm[i] = make_float2(src[i], 0.f);
    __syncthreads();
    fft_forward_stages(sm, rp.pl, rp.tw, 1, n, tid, nthr, 0, rp.pl.nstages);
    for (int i = tid; i < n; i += nthr) { const float s = tab[i]; float2 v = sm[i]; v.x *= s; v.y *= s; sm[i] = v; }
    __syncthreads();
    fft_inverse_stages(sm, rp.pl, rp.tw, 1, n, tid, nthr, 0, rp.pl.nstages);
    const float var = (mode == EPI_SNR || mode == EPI_ENVSTD) ? (float)stats[4 * row + 2] : 1.f;
    float* dst = out + row * n;
    for (int i = tid; i < n; i += nthr) dst[i] = hilbert_epilogue(sm[i], mode, var);
}

// ------------------------------------------------------------------ per-channel FFT magnitude (dsp.get_fx, dsp.py:18-38)
// one CTA per row: x[row][0:ncopy] zero-padded to n -> FFT -> out[row][(f + n/2) % n] = |X[f]| * scale (np.fft.fftshift order)
static __global__ void __launch_bounds__(256, 2)
k_row_fftmag(FftPlan pl, const float2* __restrict__ tw, const int* __restrict__ k2pos, const float* __restrict__ x, size_t ld,
             int ncopy, float scale, float* __restrict__ out) {
    extern __shared__ float2 sm[];
    const int n = pl.n, tid = threadIdx.x, nthr = blockDim.x;
    const size_t row = blockIdx.x;
    const float* src = x + row * ld;
    for (int i = tid; i < n; i += nthr) sm[i] = make_float2(i < ncopy ? src[i] : 0.f, 0.f);
    __syncthreads();
    fft_forward_stages(sm, pl, tw, 1, n, tid, nthr, 0, pl.nstages);
    float* dst = out + row * (size_t)n;
    const int half = n / 2;
    for (int j = tid; j < n; j += nthr) {
        int f = j - half; if (f < 0) f += n;                  // shifted index j holds frequency (j - n//2) mod n
        const float2 v = sm[k2pos[f]];
        dst[j] = sqrtf(v.x * v.x + v.y * v.y) * scale;
    }
}

// ------------------------------------------------------------------ forward-backward SOS IIR (scipy sosfiltfilt semantics)
constexpr int kMaxSections = 16;
struct SosParams {
    double b0[kMaxSections], b1[kMaxSections], b2[kMaxSections], a1[kMaxSections], a2[kMaxSections];
    double zi0[kMaxSections], zi1[kMaxSections];
    int nsec, pad, ns;
};

// value of the odd-extended signal at extended index e in [0, ns + 2*pad)
__device__ __forceinline__ float ext_value(const float* __restrict__ r, int e, int pad, int ns) {
    const int i = e - pad;
    if (i < 0) return 2.f * r[0] - r[-i];
    if (i >= ns) return 2.f * r[ns - 1] - r[2 * (ns - 1) - i];
    return r[i];
}

// One warp = 32 channels x one time chunk; time is walked in tiles of 32 samples staged through shared
// memory so global accesses stay coalesced while each lane runs its channel's recursion in double.
// DIR = +1: forward pass over the extended signal, writes tmp[nx][next];
// DIR = -1: backward pass over tmp, writes the central ns samples to y.
// Time chunking (chunk > 0): blockIdx.y owns extended samples [c*chunk, (c+1)*chunk) of the pass's own
// direction of travel and starts `warm` samples earlier from a zero state; the poles' decay (host picks
// warm so that |p|max^warm < 1e-9) makes the result identical to the sequential recursion at fp32
// precision.  Chunk 0 starts from SciPy's steady-state initial condition zi * first sample.
// NSEC = compile-time section count (0: generic, runtime count up to kMaxSections); NCH = time chunks a warp walks
// at once (independent recursions interleaved instruction by instruction -> twice the DFMA chains in flight per lane).
// Block = 4 warps, each warp its own (32 channels, NCH chunks) work item.
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

template <int DIR, int NSEC, int NCH>
static __global__ void __launch_bounds__(128)
k_sos_pass(SosParams sp, const float* __restrict__ x, float* __restrict__ tmp, float* __restrict__ y, int nx, int chunk,
           int warm, int nchunks) {
    // [warp][buffer][chunk][channel][time]: tiles are double-buffered -- the next 32-sample tile streams in with cp.async
    // while the recursion runs on the current one (the recursion is a dependent fp64 chain: loads must not sit in front of it)
    extern __shared__ float sos_sm[];
    typedef float Tile[32][33];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    Tile* tiles = reinterpret_cast<Tile*>(sos_sm) + (size_t)wid * 2 * NCH;      // tiles[buf * NCH + k]
    const int ch0 = (blockIdx.x * 4 + wid) * 32;
    if (ch0 >= nx) return;
    const int ns = sp.ns, pad = sp.pad, next = ns + 2 * pad;
    const int ch = ch0 + lane;
    const bool live = ch < nx;
    constexpr int NS_ = NSEC > 0 ? NSEC : kMaxSections;
    const int nsec = NSEC > 0 ? NSEC : sp.nsec;
    // progress index p = 0..next-1 along the direction of travel; extended index e = p (fwd) or next-1-p (bwd)
    int p_lo[NCH], p_hi[NCH], p_cur[NCH];
    double z0[NCH][NS_], z1[NCH][NS_];
    int steps = 0;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
        const int cidx = (int)blockIdx.y * NCH + k;
        if (chunk > 0) { p_lo[k] = cidx * chunk; p_hi[k] = min(next, p_lo[k] + chunk); }
        else { p_lo[k] = (cidx == 0) ? 0 : next; p_hi[k] = next; }
        if (cidx >= nchunks) p_lo[k] = p_hi[k] = next;                      // idle slot
        const int p_start = (chunk > 0 && cidx > 0) ? max(0, p_lo[k] - warm) : p_lo[k];
        p_cur[k] = (cidx >= nchunks) ? next : min(p_start, p_hi[k]);
        float first = 0.f;
        if (live && p_start == 0 && p_lo[k] < next) {
            if (DIR > 0) first = ext_value(x + (size_t)ch * ns, 0, pad, ns);
            else first = tmp[(size_t)ch * next + (next - 1)];
        }
#pragma unroll
        for (int s = 0; s < NS_; ++s) { z0[k][s] = sp.zi0[s] * (double)first; z1[k][s] = sp.zi1[s] * (double)first; }
        steps = max(steps, (p_hi[k] - p_cur[k] + 31) / 32);
    }
    // stage the tile that starts at progress index p0 of chunk k into buffer b (lane = progress offset, loop over channels)
    auto stage = [&](int b, int k, int p0) {
        Tile& t = tiles[b * NCH + k];
        const int p = p0 + lane;
        const bool full = (p0 + 32 <= p_hi[k]) && (nx - ch0 >= 32) && (DIR < 0 || (p0 >= pad && p0 + 32 <= pad + ns));
        if (full) {
            const float* src = (DIR > 0) ? x + (size_t)ch0 * ns + (p - pad) : tmp + (size_t)ch0 * next + (next - 1 - p);
            const size_t pitch = (DIR > 0) ? (size_t)ns : (size_t)next;
#pragma unroll 8
            for (int c = 0; c < 32; ++c) cp_async4(&t[c][lane], src + (size_t)c * pitch);
        } else {
#pragma unroll 4
            for (int c = 0; c < 32; ++c) {
                const int cc = ch0 + c;
                const int e = (DIR > 0) ? p : next - 1 - p;
                float v = 0.f;
                if (cc < nx && p < p_hi[k]) v = (DIR > 0) ? ext_value(x + (size_t)cc * ns, e, pad, ns) : tmp[(size_t)cc * next + e];
                t[c][lane] = v;
            }
        }
    };
#pragma unroll
    for (int k = 0; k < NCH; ++k) stage(0, k, p_cur[k]);
    cp_async_commit();
    for (int it = 0; it < steps; ++it) {
        const int b = it & 1;
        if (it + 1 < steps) {
#pragma unroll
            for (int k = 0; k < NCH; ++k) stage(b ^ 1, k, min(p_cur[k] + 32, p_hi[k] + 32));
        }
        cp_async_commit();
        cp_async_wait_group<1>();                 // everything but the group just committed has landed
        __syncwarp();
        if (live) {
#pragma unroll 4
            for (int q = 0; q < 32; ++q) {
                double v[NCH];
#pragma unroll
                for (int k = 0; k < NCH; ++k) v[k] = (double)tiles[b * NCH + k][lane][q];
#pragma unroll
                for (int s = 0; s < NS_; ++s) {
                    if (NSEC > 0 || s < nsec) {
#pragma unroll
                        for (int k = 0; k < NCH; ++k) {
                            const double o = fma(sp.b0[s], v[k], z0[k][s]);
                            z0[k][s] = fma(sp.b1[s], v[k], fma(-sp.a1[s], o, z1[k][s]));
                            z1[k][s] = fma(sp.b2[s], v[k], -sp.a2[s] * o);
                            v[k] = o;
                        }
                    }
                }
#pragma unroll
                for (int k = 0; k < NCH; ++k) tiles[b * NCH + k][lane][q] = (float)v[k];
            }
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < NCH; ++k) {
            const int p = p_cur[k] + lane;
            if (p >= p_lo[k] && p < p_hi[k]) {
                const int e = (DIR > 0) ? p : next - 1 - p;
#pragma unroll 8
                for (int c = 0; c < 32; ++c) {
                    const int cc = ch0 + c;
                    if (cc < nx) {
                        if (DIR > 0) tmp[(size_t)cc * next + e] = tiles[b * NCH + k][c][lane];
                        else { const int i = e - pad; if (i >= 0 && i < ns) y[(size_t)cc * ns + i] = tiles[b * NCH + k][c][lane]; }
                    }
                }
            }
            p_cur[k] = min(p_cur[k] + 32, p_hi[k] + 32);      // past p_hi: staged zeros, nothing written
        }
        __syncwarp();
    }
    cp_async_wait_group<0>();
}

// ------------------------------------------------------------------ batched STFT magnitude (librosa.stft framing)
// Frame m covers samples m*hop - nfft/2 + [0, nfft) of the zero-padded row, times the periodic
// Hann window; two frames share one complex FFT (re / im) and are untangled afterwards.
struct StftParams {
    FftPlan pl;
    const float2* tw;
    const int* k2pos;
    int nfft, hop, ns, nframes, nbins, fpb;      // fpb = frames per block (even); nbins = bins written
    int bin_lo;                                  // first DFT bin written (band slice of detect.py:390-392)
};

static __global__ void __launch_bounds__(256)
k_stft_mag(StftParams sp, const float* __restrict__ x, const float* __restrict__ win, float* __restrict__ out) {
    extern __shared__ float2 sm[];
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int n = sp.nfft, half = n / 2;
    const size_t row = blockIdx.y;
    const int m0 = blockIdx.x * sp.fpb;
    const int npair = sp.fpb / 2, fstride = n + 1;
    const float* r = x + row * sp.ns;
    for (int i = tid; i < npair * n; i += nthr) {
        const int q = i / n, j = i - q * n;
        const int ma = m0 + 2 * q, mb = ma + 1;
        const int ia = ma * sp.hop + j - half, ib = mb * sp.hop + j - half;
        const float w = win[j];
        const float a = (ma < sp.nframes && ia >= 0 && ia < sp.ns) ? r[ia] * w : 0.f;
        const float b = (mb < sp.nframes && ib >= 0 && ib < sp.ns) ? r[ib] * w : 0.f;
        sm[q * fstride + j] = make_float2(a, b);
    }
    __syncthreads();
    fft_forward_stages(sm, sp.pl, sp.tw, npair, fstride, tid, nthr, 0, sp.pl.nstages);
    float* o = out + row * (size_t)sp.nbins * sp.nframes;
    for (int i = tid; i < sp.nbins * sp.fpb; i += nthr) {
        const int kk = i / sp.fpb, f = i - kk * sp.fpb;        // frame fastest -> contiguous stores
        const int k = kk + sp.bin_lo;
        const int m = m0 + f;
        if (m >= sp.nframes) continue;
        const int q = f >> 1;
        const float2 z = sm[q * fstride + sp.k2pos[k]];
        const float2 z2 = sm[q * fstride + sp.k2pos[k == 0 ? 0 : n - k]];
        float2 v;
        if ((f & 1) == 0) v = make_float2(0.5f * (z.x + z2.x), 0.5f * (z.y - z2.y));
        else              v = make_float2(0.5f * (z.y + z2.y), 0.5f * (z2.x - z.x));
        o[(size_t)kk * sp.nframes + m] = sqrtf(v.x * v.x + v.y * v.y);
    }
}


// ------------------------------------------------------------------ sliding-DFT STFT magnitude for a band of bins
// The spectrogram-correlation detector (detect.py:650-708) asks for ~31 of the 81 bins of 160-sample frames that overlap
// by 95 % (hop 8): consecutive frames share 152 of 160 samples, and the FFT per frame above recomputes all of it.  With
// n_fft = H * P (H = hop) a frame is P blocks of H samples; per bin k
//     B_b[k]     = sum_{t<H} x[b*H + t] W^{tk}                       (block partial sum, W = exp(-2 pi i / n_fft))
//     Y_{m+1}[k] = (Y_m[k] - B_m[k] + B_{m+P}[k]) * W^{-Hk}          (rectangular-window DFT slides by one block)
//     S_m[k]     = Y_m[k]/2 - (Y_m[k-1] + Y_m[k+1])/4                (periodic Hann = three-bin combination)
// so a (frame, bin) costs one 2H-FMA block sum, one complex rotation and two complex adds.  Each thread owns one bin of one
// run of R = P*Q frames: Y is re-summed from its P blocks at the start of every run (Horner in W^{Hk}; the recursion error
// stays ~1e-6 of max|S| even for R = 240, measured in fp32 against the fp64 oracle), the last P block sums live in
// registers (the frame loop is unrolled P times so the ring index is static).  Every P frames the CTA's G runs drop their
// Y values in a shared tile from which all threads form |S| and store frame-contiguous segments.
struct SlideParams { int ns, nframes, nbins, bin_lo, nY, nYp, Q; };
constexpr int kSlideMaxThreads = 320;           // G runs x nY bins: 8 x <= 40, 16 x <= 20

// floats between the sample regions of consecutive runs: R*H + N samples + padding so that the stride is 4 (mod 32) words
// -- a warp that spans several runs then reads its (broadcast) 16-byte blocks from different banks
__host__ __device__ inline int slide_run_stride(int RH, int N) { return RH + N + ((4 - (RH + N) % 32) + 32) % 32; }

__device__ __forceinline__ float sqrt_approx(float v) {          // MUFU.SQRT, ~1 ulp, exact zero for zero
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}

template <int H>
__device__ __forceinline__ float2 slide_block(const float* __restrict__ b, const float2 (&T)[H]) {
    float xv[H];
    static_for<H / 4>([&](auto qc) {
        constexpr int q = decltype(qc)::value;
        const float4 v = *reinterpret_cast<const float4*>(b + 4 * q);
        xv[4 * q] = v.x; xv[4 * q + 1] = v.y; xv[4 * q + 2] = v.z; xv[4 * q + 3] = v.w;
    });
    float re = xv[0], im = 0.f;                 // T[0] = 1
    static_for<H - 1>([&](auto tc) {
        constexpr int t = decltype(tc)::value + 1;
        re = fmaf(xv[t], T[t].x, re);
        im = fmaf(xv[t], T[t].y, im);
    });
    return make_float2(re, im);
}

template <int H, int P, int G>
static __global__ void __launch_bounds__(kSlideMaxThreads, 2)
k_stft_slide(SlideParams sp, const float* __restrict__ x, const float2* __restrict__ wn, float* __restrict__ out) {
    constexpr int N = H * P;
    extern __shared__ __align__(16) float sl_smem[];
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int R = P * sp.Q, nY = sp.nY, nYp = sp.nYp;
    const int RL = R * H + N, RS = slide_run_stride(R * H, N);      // samples of one run (its R frames + one block), stride
    float* xs = sl_smem;                                             // [G][RS]
    float2* Yt = reinterpret_cast<float2*>(sl_smem + G * RS);        // [G][P][nYp]
    const size_t row = blockIdx.y;
    const int M0 = blockIdx.x * G * R;
    const float* r = x + row * (size_t)sp.ns;
    for (int gg = 0; gg < G; ++gg) {
        const long long s0 = (long long)(M0 + gg * R) * H - N / 2;
        float* dst = xs + gg * RS;
        for (int i = tid; i < RL; i += nthr) {
            const long long s = s0 + i;
            dst[i] = (s >= 0 && s < sp.ns) ? r[s] : 0.f;
        }
    }
    const int g = tid / nY, kk = tid - g * nY;
    const bool act = g < G;
    float2 T[H], w;
    {
        int k = (sp.bin_lo - 1 + kk) % N;
        if (k < 0) k += N;                                           // bin -1 is bin N-1; no special case for the edges
        static_for<H>([&](auto tc) { constexpr int t = decltype(tc)::value; T[t] = wn[(t * k) % N]; });
        w = wn[(H * k) % N];
    }
    __syncthreads();
    const float* xb = xs + (size_t)(act ? g : 0) * RS;
    float2 ring[P], Y = make_float2(0.f, 0.f);
    static_for<P>([&](auto ic) {
        constexpr int p = P - 1 - decltype(ic)::value;
        ring[p] = slide_block<H>(xb + p * H, T);
        Y = make_float2(fmaf(Y.x, w.x, fmaf(-Y.y, w.y, ring[p].x)), fmaf(Y.x, w.y, fmaf(Y.y, w.x, ring[p].y)));
    });
    float* orow = out + row * (size_t)sp.nbins * sp.nframes;
    for (int q = 0; q < sp.Q; ++q) {
        if (act) {
            float2* yt = Yt + (size_t)(g * P) * nYp + kk;
            const float* xq = xb + (size_t)(q * P + P) * H;          // block entering after local frame q*P + j
            static_for<P>([&](auto jc) {
                constexpr int j = decltype(jc)::value;
                yt[j * nYp] = Y;
                const float2 E = slide_block<H>(xq + j * H, T);
                const float dx = Y.x - ring[j].x + E.x, dy = Y.y - ring[j].y + E.y;
                Y = make_float2(fmaf(dx, w.x, dy * w.y), fmaf(dy, w.x, -dx * w.y));      // times conj(w) = W^{-Hk}
                ring[j] = E;
            });
        }
        __syncthreads();
        // |S|: each thread walks half of the band of one frame with a three-bin window (one 8-byte read per output)
        const int mq = M0 + q * P, nh = (sp.nbins + 1) >> 1;
        for (int it = tid; it < 2 * G * P; it += nthr) {
            const int half = it / (G * P), pr = it - half * (G * P);             // pr = run * P + frame of the sub-step
            const int gg = pr / P, fl = pr - gg * P;
            const int m = mq + gg * R + fl;
            if (m >= sp.nframes) continue;
            const int o0 = half * nh, o1 = min(sp.nbins, o0 + nh);
            const float2* y = Yt + (size_t)pr * nYp + o0;
            float* po = orow + (size_t)o0 * sp.nframes + m;
            float2 a = y[0], b = y[1];
#pragma unroll 4
            for (int o = o0; o < o1; ++o) {
                const float2 c = y[o - o0 + 2];
                const float re = 0.5f * b.x - 0.25f * (a.x + c.x), im = 0.5f * b.y - 0.25f * (a.y + c.y);
                *po = sqrt_approx(fmaf(re, re, im * im));
                po += sp.nframes; a = b; b = c;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------ per-row median of non-negative floats
// np.median over each row (detect.xcorr2d divides by median(spectro), detect.py:600), exact.  Even counts average the
// two middle order statistics.
//   select_rank: 3-pass radix select on the float bit patterns (monotone for x >= 0): 11 + 11 + 10 bits.
//   k_row_median: rows longer than the shared buffer are bracketed first -- m = 2048 .. 16 384 evenly spaced samples are
//   sorted in shared memory, the values 1.375 sqrt(m) sample ranks (2.75 sigma of a quantile's sample rank) either side of
//   the median's position bound it with ~99 % probability, ONE pass over the row counts what lies below the bracket and collects what
//   lies inside (~2 % of the row) in shared memory, and the radix select runs on that.  If the bracket misses (or ties
//   overflow the buffer) the row falls back to the radix select over global memory, so the result never depends on luck.
constexpr int kMedThreads = 512, kMedCap = 16384;

// bin holding `rank` in hist[nb] (nb = 1024 or 2048) by a block-wide scan; returns (bin, rank inside the bin) to all threads
__device__ __forceinline__ void find_bin(const unsigned int* hist, int nb, unsigned long long rank, unsigned int& bin, unsigned long long& rin) {
    __shared__ unsigned int ws[kMedThreads / 32];
    __shared__ unsigned int s_bin;
    __shared__ unsigned long long s_rank;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int per = nb / kMedThreads;
    unsigned int c[4] = {0, 0, 0, 0}, tsum = 0;
    for (int i = 0; i < per; ++i) { c[i] = hist[tid * per + i]; tsum += c[i]; }
    unsigned int inc = tsum;
    for (int d = 1; d < 32; d <<= 1) { const unsigned int v = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += v; }
    if (lane == 31) ws[wid] = inc;
    __syncthreads();
    unsigned long long excl = inc - tsum;
    for (int w = 0; w < wid; ++w) excl += ws[w];
    if (tsum > 0 && rank >= excl && rank < excl + tsum) {
        unsigned long long acc = excl;
        int i = 0;
        for (; i < per - 1; ++i) { if (acc + c[i] > rank) break; acc += c[i]; }
        s_bin = (unsigned int)(tid * per + i); s_rank = rank - acc;
    }
    __syncthreads();
    bin = s_bin; rin = s_rank;
    __syncthreads();
}

__device__ __forceinline__ unsigned int select_rank(const float* __restrict__ r, size_t n, size_t rank, unsigned int* hist) {
    unsigned int prefix = 0, mask = 0;
    const int shifts[3] = {21, 10, 0};
    const int bits[3] = {11, 11, 10};
    for (int pass = 0; pass < 3; ++pass) {
        const int nb = 1 << bits[pass];
        for (int i = threadIdx.x; i < nb; i += blockDim.x) hist[i] = 0;
        __syncthreads();
        for (size_t i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned int u = __float_as_uint(r[i]);
            if ((u & mask) == prefix) atomicAdd(&hist[(u >> shifts[pass]) & (nb - 1)], 1u);
        }
        __syncthreads();
        unsigned int bin; unsigned long long rin;
        find_bin(hist, nb, rank, bin, rin);
        prefix |= bin << shifts[pass];
        mask |= (unsigned int)(nb - 1) << shifts[pass];
        rank = (size_t)rin;
    }
    return prefix;
}

// row r is the n values from x + r * ld (ld >= n): ld = n for a dense matrix, ld > n for a band of rows of a spectrogram
static __global__ void __launch_bounds__(kMedThreads)
k_row_median(const float* __restrict__ x, size_t n, size_t ld, float* __restrict__ med) {
    extern __shared__ __align__(16) float mbuf[];                // kMedCap floats: samples, then the bracket's contents
    __shared__ unsigned int hist[2048];
    __shared__ unsigned int s_cnt;
    __shared__ unsigned long long s_below[kMedThreads / 32];
    __shared__ float s_lohi[2];
    const int tid = threadIdx.x, lane = tid & 31;
    const float* r = x + (size_t)blockIdx.x * ld;
    const size_t rk_hi = n / 2, rk_lo = (n & 1) ? n / 2 : n / 2 - 1;
    const float* src = r;                                        // where the final select runs
    size_t cnt = n, below = 0;
    if (n <= (size_t)kMedCap) {
        for (size_t i = tid; i < n; i += kMedThreads) mbuf[i] = r[i];
        __syncthreads();
        src = mbuf;
    } else {
        // smallest sample (the sort is the expensive part) whose +-2.75 sigma bracket, ~2.75 n / sqrt(m) entries, fits 90 % of
        // the buffer: n <= 0.9 * 16384 * sqrt(m) / 2.75
        int m = 2048;
        while (m < kMedCap && (double)n > 5362.0 * sqrt((double)m)) m <<= 1;
        for (int i = tid; i < m; i += kMedThreads) mbuf[i] = r[(size_t)(((unsigned long long)i * n + n / 2) / m)];
        __syncthreads();
        for (int k = 2; k <= m; k <<= 1)                         // bitonic sort, ascending; one compare-exchange per pair
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int pi = tid; pi < (m >> 1); pi += kMedThreads) {
                    const int i = ((pi & ~(j - 1)) << 1) | (pi & (j - 1)), l = i | j;
                    const float a = mbuf[i], b = mbuf[l];
                    if (((i & k) == 0) ? (a > b) : (a < b)) { mbuf[i] = b; mbuf[l] = a; }
                }
                __syncthreads();
            }
        if (tid == 0) {
            // 2.75 sigma of a quantile's sample rank (sigma = sqrt(m) / 2), shrunk if the bracket would not fit the buffer
            long long delta = (long long)(1.375 * sqrt((double)m));
            const long long fit = (long long)(0.45 * (double)kMedCap * (double)m / (double)n);
            if (delta > fit) delta = fit > 1 ? fit : 1;
            const long long ps = (long long)(((unsigned long long)rk_hi * m) / n);
            s_lohi[0] = mbuf[max(0LL, ps - delta)];
            s_lohi[1] = mbuf[min((long long)m - 1, ps + delta)];
            s_cnt = 0;
        }
        __syncthreads();
        const float lo = s_lohi[0], hi = s_lohi[1];
        __syncthreads();                                         // everyone holds lo / hi before the buffer is reused
        unsigned long long nb_ = 0;
        for (size_t i0 = 0; i0 < n; i0 += 4 * kMedThreads) {
            float v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {                        // entries are >= 0: -1 is outside every bracket
                const size_t i = i0 + u * kMedThreads + tid;
                v[u] = i < n ? r[i] : -1.f;
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const bool ok = v[u] >= 0.f;
                nb_ += (ok && v[u] < lo) ? 1u : 0u;
                const bool in = ok && v[u] >= lo && v[u] <= hi;
                const unsigned int bal = __ballot_sync(0xffffffffu, in);
                if (bal) {
                    unsigned int base = 0;
                    if (lane == 0) base = atomicAdd(&s_cnt, (unsigned int)__popc(bal));
                    base = __shfl_sync(0xffffffffu, base, 0);
                    const unsigned int pos = base + __popc(bal & ((1u << lane) - 1u));
                    if (in && pos < (unsigned int)kMedCap) mbuf[pos] = v[u];
                }
            }
        }
        for (int d = 16; d > 0; d >>= 1) nb_ += __shfl_down_sync(0xffffffffu, nb_, d);
        if (lane == 0) s_below[tid >> 5] = nb_;
        __syncthreads();
        for (int w = 0; w < kMedThreads / 32; ++w) below += (size_t)s_below[w];
        cnt = s_cnt;
        if (cnt <= (size_t)kMedCap && rk_lo >= below && rk_hi < below + cnt) src = mbuf;
        else { below = 0; cnt = n; }                             // bracket missed or overflowed: select over the whole row
        __syncthreads();
    }
    const float vhi = __uint_as_float(select_rank(src, cnt, rk_hi - below, hist));
    float vlo = vhi;
    if (rk_lo != rk_hi) vlo = __uint_as_float(select_rank(src, cnt, rk_lo - below, hist));
    if (tid == 0) med[blockIdx.x] = 0.5f * (vlo + vhi);
}

// ------------------------------------------------------------------ spectrogram x kernel correlation (detect.xcorr2d)
// out[row][t] = max(0, sum_f sum_j S[row][f][t - c0 + j] * K[f][j]) / (median[row] * kw),  c0 = ceil((kw-1)/2)
// = fftconvolve(S, flip(K, axis=1), 'same', axes=1).sum(0), clipped and normalised (detect.py:597-600).
static __global__ void __launch_bounds__(256)
k_speccorr(const float* __restrict__ S, int nf, int nt, const float* __restrict__ K, int kw, const float* __restrict__ med,
           float* __restrict__ out) {
    extern __shared__ float sh[];
    float* sk = sh;                          // [nf][kw]
    float* st = sh + nf * kw;                // [nf][tile + kw]
    const int tile = blockDim.x, w = tile + kw;
    const size_t row = blockIdx.y;
    const int t0 = blockIdx.x * tile;
    const int c0 = kw / 2;                   // ceil((kw-1)/2)
    for (int i = threadIdx.x; i < nf * kw; i += blockDim.x) sk[i] = K[i];
    const float* Sr = S + row * (size_t)nf * nt;
    for (int i = threadIdx.x; i < nf * w; i += blockDim.x) {
        const int f = i / w, j = i - f * w;
        const int t = t0 - c0 + j;
        st[i] = (t >= 0 && t < nt) ? Sr[(size_t)f * nt + t] : 0.f;
    }
    __syncthreads();
    const int t = t0 + threadIdx.x;
    if (t >= nt) return;
    float acc = 0.f;
    for (int f = 0; f < nf; ++f) {
        const float* a = st + f * w + threadIdx.x;
        const float* b = sk + f * kw;
        for (int j = 0; j < kw; ++j) acc = fmaf(a[j], b[j], acc);
    }
    acc = fmaxf(acc, 0.f);
    out[row * nt + t] = acc / (med[row] * (float)kw);
}

// Register-tiled version (default): four consecutive outputs per thread, the time window slides through two float4
// registers and the kernel row arrives as broadcast float4 -- 2 shared loads per 16 FMAs instead of 2 per FMA.
// Several kernels share one staged tile: S holds nfs frequency rows per channel, the rows fs0 .. fs0 + nst - 1 (the union
// of the kernels' bands) are staged once, and kernel k reads its nf[k] rows from staged row f0[k].  Every kernel gets
// pad[k] = c0 - kw[k] / 2 leading zeros up to the common centre c0 = max kw / 2, so all of them read the same window
// t - c0 ..; a zero product leaves the fp32 sum unchanged and each kernel keeps its f-ascending, j-ascending order, so
// every output is bit-equal to a one-kernel launch (and to k_speccorr).
// Shared layout: sk_k [nf[k]][kwp] for each k (padded kernel rows, kwp = multiple of 4), st [nst][w], w = 4 * threads + kwp.
constexpr int kScThreads = 128, kScTile = 4 * kScThreads, kScMaxKernels = 8;

struct SpecCorrSet {
    const float* K[kScMaxKernels];            // [nf][kw] each
    const float* med[kScMaxKernels];          // [nx] each
    float* out[kScMaxKernels];                // [nx][nt] each
    int f0[kScMaxKernels], nf[kScMaxKernels], kw[kScMaxKernels], pad[kScMaxKernels];
    int nk, nfs, fs0, nst, c0, kwp;
};

static __global__ void __launch_bounds__(kScThreads)
k_speccorr4(const float* __restrict__ S, int nt, const __grid_constant__ SpecCorrSet set) {
    extern __shared__ __align__(16) float sh4[];
    const int kwp = set.kwp, nst = set.nst, c0 = set.c0;
    const int w = kScTile + kwp;
    const int tid = threadIdx.x;
    const size_t row = blockIdx.y;
    const int t0 = blockIdx.x * kScTile;
    float* st = sh4;                                             // [nst][w] after the kernels
#pragma unroll 1
    for (int k = 0; k < set.nk; ++k) {
        const float* K = set.K[k];
        const int kw = set.kw[k], pad = set.pad[k], n = set.nf[k] * kwp;
        for (int i = tid; i < n; i += kScThreads) {
            const int f = i / kwp, j = i - f * kwp - pad;
            st[i] = (j >= 0 && j < kw) ? K[f * kw + j] : 0.f;
        }
        st += n;
    }
    const float* Sr = S + row * (size_t)set.nfs * nt + (size_t)set.fs0 * nt;
    const int fq = (nst + 3) >> 2;                               // frequency rows per staging group
#pragma unroll 1
    for (int gq = 0; gq < 4; ++gq) {
        const int f0 = gq * fq, f1 = min(nst, f0 + fq);
        for (int j = tid; j < w; j += kScThreads) {              // column first: bounds and addresses once per column
            const int t = t0 - c0 + j;
            float* dst = st + f0 * w + j;
            if (t >= 0 && t < nt) {
                const float* src = Sr + (size_t)f0 * nt + t;
#pragma unroll 4
                for (int f = f0; f < f1; ++f, dst += w, src += nt) cp_async4(dst, src);
            } else {
#pragma unroll 1
                for (int f = f0; f < f1; ++f, dst += w) *dst = 0.f;
            }
        }
        cp_async_commit();
    }
    const int nq = kwp >> 2;
    const float* sk = sh4;
#pragma unroll 1
    for (int k = 0; k < set.nk; ++k) {                           // kernel 0 overlaps the staging; the others find it landed
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        auto mac16 = [&](const float4& lo, const float4& hi, const float4& kv) {
            const float win[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
            const float kk[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
            for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                for (int oo = 0; oo < 4; ++oo) acc[oo] = fmaf(win[jj + oo], kk[jj], acc[oo]);
        };
        const int fa = set.f0[k], fb = fa + set.nf[k];
#pragma unroll 1                                             // one copy of the FMA block: unrolled four times it missed the i-cache
        for (int gq = 0; gq < 4; ++gq) {
            if (k == 0) {
                if (gq == 0) cp_async_wait_group<3>(); else if (gq == 1) cp_async_wait_group<2>();
                else if (gq == 2) cp_async_wait_group<1>(); else cp_async_wait_group<0>();
                __syncthreads();
            }
#pragma unroll 1
            for (int f = max(fa, gq * fq); f < min(fb, (gq + 1) * fq); ++f) {
                const float4* a = reinterpret_cast<const float4*>(st + f * w) + tid;
                const float4* b = reinterpret_cast<const float4*>(sk + (f - fa) * kwp);
                float4 c0v = a[0], c1v;
                int q = 0;
#pragma unroll 1
                for (; q + 1 < nq; q += 2) {                     // the window ping-pongs between two registers: no moves
                    c1v = a[q + 1]; mac16(c0v, c1v, b[q]);
                    c0v = a[q + 2]; mac16(c1v, c0v, b[q + 1]);
                }
                if (q < nq) { c1v = a[q + 1]; mac16(c0v, c1v, b[q]); }
            }
        }
        const float den = set.med[k][row] * (float)set.kw[k];  // same expression as the untiled kernel: identical rounding
        float* out = set.out[k];
#pragma unroll
        for (int oo = 0; oo < 4; ++oo) {
            const int t = t0 + 4 * tid + oo;
            if (t < nt) out[row * nt + t] = fmaxf(acc[oo], 0.f) / den;
        }
        sk += set.nf[k] * kwp;
    }
}

// per-row maximum (spectrogram normalisation max(S) of dsp.py:76 / detect.py:387)
static __global__ void __launch_bounds__(256)
k_row_max(const float* __restrict__ x, size_t n, float* __restrict__ mx) {
    __shared__ float s[8];
    const float* r = x + (size_t)blockIdx.x * n;
    float m = 0.f;
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, r[i]);
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) { for (int w = 1; w < 8; ++w) m = fmaxf(m, s[w]); mx[blockIdx.x] = fmaxf(m, s[0]); }
}


// ------------------------------------------------------------------ peak picking: find_peaks(x, prominence >= thr)
// Semantics of scipy.signal.find_peaks as called by detect.pick_times_env / pick_times (detect.py:192, :271):
//  * local maxima incl. flat tops: i is a plateau start if x[i-1] < x[i]; with e the first index > i whose value
//    differs (at most n-1), it is a peak iff x[e] < x[i]; the reported index is (i + e - 1) / 2; never index 0 / n-1;
//  * prominence = x[p] - max(left_min, right_min) where each side is the minimum over the run of samples <= x[p]
//    adjacent to p (the run ends at the first strictly greater sample or the array end); compared in double.
// The runs are walked hierarchically (64-sample blocks, 64-block superblocks with precomputed max / min), so a peak
// costs O(64 * 3) reads in the worst case instead of O(n).
constexpr int kPkB = 64;

struct PeakLevels { const float *bmax, *bmin, *smax, *smin; int nb1, nb2; };

static __global__ void __launch_bounds__(256)
k_peak_levels(const float* __restrict__ x, int ns, float* bmax, float* bmin, float* smax, float* smin, float* rowmin, int nb1, int nb2) {
    const size_t row = blockIdx.x;
    const float* r = x + row * (size_t)ns;
    float* bm = bmax + row * nb1; float* bn = bmin + row * nb1;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int b = wid; b < nb1; b += nw) {
        const int i0 = b * kPkB + 2 * lane;
        float mx = -INFINITY, mn = INFINITY;
        if (i0 < ns) { const float v = r[i0]; mx = v; mn = v; }
        if (i0 + 1 < ns) { const float v = r[i0 + 1]; mx = fmaxf(mx, v); mn = fminf(mn, v); }
        for (int o = 16; o; o >>= 1) { mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o)); mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o)); }
        if (lane == 0) { bm[b] = mx; bn[b] = mn; }
    }
    __syncthreads();
    for (int sb = threadIdx.x; sb < nb2; sb += blockDim.x) {
        float mx = -INFINITY, mn = INFINITY;
        for (int b = sb * kPkB; b < min(nb1, (sb + 1) * kPkB); ++b) { mx = fmaxf(mx, bm[b]); mn = fminf(mn, bn[b]); }
        smax[row * nb2 + sb] = mx; smin[row * nb2 + sb] = mn;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float mn = INFINITY;
        for (int sb = 0; sb < nb2; ++sb) mn = fminf(mn, smin[row * nb2 + sb]);
        rowmin[row] = mn;
    }
}

// minimum over the run of samples <= v adjacent to position p on one side (DIR = -1 left, +1 right), v included
template <int DIR>
__host__ __device__ __forceinline__ float peak_side_min(const float* __restrict__ r, int ns, int p, float v, const float* __restrict__ bm,
                                               const float* __restrict__ bn, const float* __restrict__ sm, const float* __restrict__ sn,
                                               int nb1) {
    float m = v;
    int b = p / kPkB;
    // rest of p's own block
    if (DIR < 0) { for (int i = p - 1; i >= b * kPkB; --i) { const float u = r[i]; if (u > v) return m; m = fminf(m, u); } }
    else { const int e = ns < (b + 1) * kPkB ? ns : (b + 1) * kPkB; for (int i = p + 1; i < e; ++i) { const float u = r[i]; if (u > v) return m; m = fminf(m, u); } }
    b += DIR;
    while (b >= 0 && b < nb1) {
        const int sb = b / kPkB;
        const bool sb_edge = DIR < 0 ? (b % kPkB == kPkB - 1) : (b % kPkB == 0);
        const bool sb_full = DIR < 0 ? true : ((sb + 1) * kPkB <= nb1);
        if (sb_edge && sb_full && !(sm[sb] > v)) { m = fminf(m, sn[sb]); b += DIR * kPkB; continue; }    // whole superblock <= v
        if (!(bm[b] > v)) { m = fminf(m, bn[b]); b += DIR; continue; }                                   // whole block <= v
        const int lo = b * kPkB, hi = ns < lo + kPkB ? ns : lo + kPkB;
        if (DIR < 0) { for (int i = hi - 1; i >= lo; --i) { const float u = r[i]; if (u > v) return m; m = fminf(m, u); } }
        else { for (int i = lo; i < hi; ++i) { const float u = r[i]; if (u > v) return m; m = fminf(m, u); } }
        b += DIR;                                          // only reached when the block's maximum is a NaN artefact
    }
    return m;
}

// index of the accepted peak whose flat top starts at sample i, or -1 (one call per sample; shared by the kernel and
// the host emulation test)
__host__ __device__ __forceinline__ int peak_pick_one(const float* __restrict__ r, int ns, int i, const float* __restrict__ bm,
                                                      const float* __restrict__ bn, const float* __restrict__ sm,
                                                      const float* __restrict__ sn, int nb1, float rowmin, double thr) {
    if (i < 1 || i >= ns - 1) return -1;
    const float v = r[i];
    if (!(r[i - 1] < v)) return -1;
    int e = i + 1;
    while (e < ns - 1 && r[e] == v) ++e;
    if (!(r[e] < v)) return -1;
    if ((double)v - (double)rowmin < thr) return -1;                   // prominence <= height above the row minimum
    const int p = (i + e - 1) / 2;
    const float lmin = peak_side_min<-1>(r, ns, p, v, bm, bn, sm, sn, nb1);
    const float rmin = peak_side_min<+1>(r, ns, p, v, bm, bn, sm, sn, nb1);
    return ((double)v - (double)fmaxf(lmin, rmin) >= thr) ? p : -1;
}

static __global__ void __launch_bounds__(256)
k_peak_pick(const float* __restrict__ x, int ns, PeakLevels lv, const float* __restrict__ rowmin, double thr, unsigned char* __restrict__ flags) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t row = blockIdx.y;
    if (i >= ns) return;
    const int p = peak_pick_one(x + row * (size_t)ns, ns, i, lv.bmax + row * lv.nb1, lv.bmin + row * lv.nb1, lv.smax + row * lv.nb2,
                                lv.smin + row * lv.nb2, lv.nb1, rowmin[row], thr);
    if (p >= 0) flags[row * (size_t)ns + p] = 1;
}

// ------------------------------------------------------------------ loader-side fusion: raw counts -> strain
// data_handle.raw2strain (data_handle.py:157-177): trace -= mean(trace, axis=1); trace *= scale_factor, here straight from
// the on-disk int32 (or float32) counts to fp32 strain; one CTA per channel, mean accumulated in double.
template <typename T>
static __global__ void __launch_bounds__(512)
k_raw2strain(const T* __restrict__ raw, float* __restrict__ out, int ns, double scale) {
    const size_t row = blockIdx.x;
    const T* r = raw + row * (size_t)ns;
    float* o = out + row * (size_t)ns;
    const bool vec = (ns % 4 == 0) && (((size_t)r | (size_t)o) % 16 == 0);
    using V4 = typename std::conditional<std::is_same<T, int>::value, int4, float4>::type;
    double acc = 0.0;
    if (vec) {
        const V4* r4 = reinterpret_cast<const V4*>(r);
        for (int i = threadIdx.x; i < ns / 4; i += blockDim.x) { const V4 v = r4[i]; acc += ((double)v.x + (double)v.y) + ((double)v.z + (double)v.w); }
    } else {
        for (int i = threadIdx.x; i < ns; i += blockDim.x) acc += (double)r[i];
    }
    __shared__ double s_part[16];
    for (int o2 = 16; o2; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    double mean = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) mean += s_part[w];
    mean /= (double)ns;
    if (vec) {                                               // second read of the row comes from L2
        const V4* r4 = reinterpret_cast<const V4*>(r);
        float4* o4 = reinterpret_cast<float4*>(o);
        for (int i = threadIdx.x; i < ns / 4; i += blockDim.x) {
            const V4 v = r4[i];
            o4[i] = make_float4((float)(((double)v.x - mean) * scale), (float)(((double)v.y - mean) * scale),
                                (float)(((double)v.z - mean) * scale), (float)(((double)v.w - mean) * scale));
        }
    } else {
        for (int i = threadIdx.x; i < ns; i += blockDim.x) o[i] = (float)(((double)r[i] - mean) * scale);
    }
}

}  // namespace d4w
