// welch_kernels.cuh -- Welch power spectral density of row chunks (d4w_welch, d4w_welch.cu), the per-chunk
// scipy.signal.welch of tools.spec / tools.__spec_chunk (das4whales/tools.py:212-236).
//
// One CTA per (row, chunk).  Segment s of a chunk is samples [s * step, s * step + nperseg), nseg = (chunk - nperseg) / step
// + 1 (SciPy drops a trailing partial segment).  Segments go through the shared-memory FFT engine in batches of up to
// 2 * kWelchMaxPairs, two real segments per complex nfft-point frame (re / im), untangled afterwards as k_stft_mag does:
//   stage     frame q <- segments 2q, 2q+1 of the batch, zero-padded to nfft (an odd last segment gets a zero partner)
//   detrend   'constant': each segment's mean (double, fixed summation order) is subtracted, then the window multiplies
//   FFT       fft_forward_stages over the batch's frames
//   untangle  |X_k|^2 for the one-sided bins k = 0 .. nfft/2, times scale and SciPy's one-sided doubling (every bin but DC
//             and, for even nfft, Nyquist).  Bin k is read at k2pos[k], the position map of the stages in `pl` (for
//             n = 2520 the d4w_fft_plan's own table is the prime-factor map of the matched filter, so d4w_welch passes
//             another one)
//   average   mean: summed in double in segment order in shared memory, divided by nseg at the end;
//             median in shared memory (nseg <= kWelchSmemMedianSeg and every periodogram fits the budget): exact rank selection per
//             bin, the two middle order statistics averaged for even nseg, as k_row_median does;
//             median through the workspace: periodograms written bin-major, ws[(block * nbins + k) * nseg + s], for
//             d4w_row_median.
// For the median the periodograms are scaled by 1 / _median_bias(nseg) before the selection; the scaling is monotone, so
// the selected order statistics are those of the unscaled values.
//
// The body is __host__ __device__ with (block, tid, nthr, smem) loops, so that tests/host_emul/welch_emul.cu runs it block
// by block on the CPU.
#pragma once
#include <algorithm>
#include "fft_smem.cuh"

namespace d4w {

constexpr int kWelchThreads = 256;
constexpr int kWelchMaxPairs = 4;              // complex frames per FFT batch (8 segments)
// Rank selection in shared memory costs nseg^2 compares per bin and thread: on an H100, 92 segments of nperseg 256 at
// 11 020 x 12 000 took 9.0 ms more than the mean.  The workspace route adds a d4w_row_median CTA per (row, bin): 54.5 ms for
// 5.1 million 233-value rows, so ~15 ms for those 1.4 million.  The quadratic cost crosses it near 120 segments (DESIGN §4).
constexpr int kWelchSmemMedianSeg = 112;
constexpr size_t kWelchSmemBudget = 100 * 1024; // two CTAs per SM

enum { kWelchMean = 0, kWelchMedianSmem = 1, kWelchMedianWs = 2 };

struct WelchParams {
    FftPlan pl;
    const float2* tw;
    const int* k2pos;            // DFT bin -> position after the forward stages of pl
    int nfft, nperseg, step, ns, chunk, nchunks, nseg, nbins;
    int pairs;                   // complex frames per batch
    int fstride;                 // float2 between frames (odd for even nfft)
    int detrend;                 // 1: subtract each segment's mean
    int mode;                    // kWelchMean / kWelchMedianSmem / kWelchMedianWs
    double scale;                // SciPy's scale, divided by nseg (mean) or by _median_bias(nseg) (median)
};

__host__ __device__ inline int welch_fstride(int nfft) { return nfft + (nfft % 2 == 0 ? 1 : 0); }

// shared-memory layout of one CTA: [partial sums: kWelchThreads doubles][bin sums: nbins doubles (mean)]
// [frames: pairs x fstride float2][periodograms: nseg x nbins floats (median in shared memory)][segment means: 2 x pairs]
__host__ __device__ inline size_t welch_smem_bytes(int nfft, int nbins, int nseg, int pairs, int mode) {
    return (size_t)kWelchThreads * sizeof(double) + (mode == kWelchMean ? (size_t)nbins * sizeof(double) : 0) +
           (size_t)pairs * welch_fstride(nfft) * sizeof(float2) + (mode == kWelchMedianSmem ? (size_t)nseg * nbins * sizeof(float) : 0) +
           (size_t)2 * kWelchMaxPairs * sizeof(float);
}

// SciPy's _median_bias(n): 1 + sum_{i=1}^{(n-1)/2} (1 / (2i + 1) - 1 / (2i))
inline double welch_median_bias(int n) {
    double s = 0.0;
    for (int i = 1; i <= (n - 1) / 2; ++i) s += 1.0 / (2.0 * i + 1.0) - 1.0 / (2.0 * i);
    return 1.0 + s;
}

// Geometry, averaging route and batch size.  Returns 0, or 1 when one frame pair does not fit `smem_cap` (the nfft limit);
// `smem` is the CTA's shared memory.  Sizes must already be valid (d4w_welch checks them).
inline int welch_config(const FftPlan& pl, int ns, int chunk, int nperseg, int step, int detrend, double scale, int median,
                        size_t smem_cap, WelchParams& wp, size_t& smem) {
    wp = WelchParams{};
    wp.pl = pl;
    wp.nfft = pl.n; wp.nperseg = nperseg; wp.step = step; wp.ns = ns; wp.chunk = chunk;
    wp.nchunks = ns / chunk;
    wp.nseg = (chunk - nperseg) / step + 1;
    wp.nbins = pl.n / 2 + 1;
    wp.fstride = welch_fstride(pl.n);
    wp.detrend = detrend ? 1 : 0;
    wp.mode = !median ? kWelchMean
            : (wp.nseg <= kWelchSmemMedianSeg &&
               welch_smem_bytes(pl.n, wp.nbins, wp.nseg, 1, kWelchMedianSmem) <= kWelchSmemBudget) ? kWelchMedianSmem
            : kWelchMedianWs;
    wp.scale = median ? scale / welch_median_bias(wp.nseg) : scale / wp.nseg;
    const int want = std::min(kWelchMaxPairs, (wp.nseg + 1) / 2);
    wp.pairs = 1;
    while (wp.pairs < want && welch_smem_bytes(pl.n, wp.nbins, wp.nseg, wp.pairs + 1, wp.mode) <= kWelchSmemBudget) ++wp.pairs;
    smem = welch_smem_bytes(pl.n, wp.nbins, wp.nseg, wp.pairs, wp.mode);
    return smem <= smem_cap ? 0 : 1;
}

// One (row, chunk) = `block`.  x: [nrows][ns]; out: [nrows][nchunks][nbins]; ws: the bin-major periodograms (kWelchMedianWs).
__host__ __device__ inline void welch_body(const WelchParams& wp, const float* __restrict__ x, const float* __restrict__ win,
                                           float* __restrict__ out, float* __restrict__ ws, long long block, int tid, int nthr,
                                           void* smem) {
    double* part = static_cast<double*>(smem);                                      // [kWelchThreads]
    double* sums = part + kWelchThreads;                                            // [nbins] (mean)
    float2* fr = reinterpret_cast<float2*>(sums + (wp.mode == kWelchMean ? wp.nbins : 0));
    float* per = reinterpret_cast<float*>(fr + (size_t)wp.pairs * wp.fstride);      // [nseg][nbins] (median in smem)
    float* mu = per + (wp.mode == kWelchMedianSmem ? (size_t)wp.nseg * wp.nbins : 0);  // [2 * kWelchMaxPairs]
    const long long row = block / wp.nchunks;
    const int c = (int)(block - row * wp.nchunks);
    const float* xr = x + (size_t)row * wp.ns + (size_t)c * wp.chunk;
    const int n = wp.nfft, L = wp.nperseg, fst = wp.fstride, nbins = wp.nbins;
    const int batch = 2 * wp.pairs;
    const int G = nthr / batch > 0 ? nthr / batch : 1;                              // partial sums per segment mean
    if (wp.mode == kWelchMean)
        for (int k = tid; k < nbins; k += nthr) sums[k] = 0.0;
    for (int s0 = 0; s0 < wp.nseg; s0 += batch) {
        const int cnt = wp.nseg - s0 < batch ? wp.nseg - s0 : batch;                // segments in this batch
        const int npair = (cnt + 1) / 2;
        for (int i = tid; i < npair * n; i += nthr) {
            const int q = i / n, j = i - q * n;
            float a = 0.f, b = 0.f;
            if (j < L) {
                a = xr[(size_t)(s0 + 2 * q) * wp.step + j];
                if (2 * q + 1 < cnt) b = xr[(size_t)(s0 + 2 * q + 1) * wp.step + j];
            }
            fr[q * fst + j] = make_float2(a, b);
        }
        D4W_SYNC();
        if (wp.detrend) {
            for (int id = tid; id < batch * G; id += nthr) {
                const int sg = id / G, l = id - sg * G;
                double acc = 0.0;
                if (sg < cnt) {
                    const float* f = reinterpret_cast<const float*>(fr + (size_t)(sg >> 1) * fst) + (sg & 1);
                    for (int j = l; j < L; j += G) acc += (double)f[2 * j];
                }
                part[id] = acc;
            }
            D4W_SYNC();
            for (int sg = tid; sg < batch; sg += nthr) {
                double acc = 0.0;
                for (int l = 0; l < G; ++l) acc += part[sg * G + l];
                mu[sg] = sg < cnt ? (float)(acc / L) : 0.f;
            }
            D4W_SYNC();
        }
        for (int i = tid; i < npair * L; i += nthr) {
            const int q = i / L, j = i - q * L;
            float2 v = fr[q * fst + j];
            if (wp.detrend) { v.x -= mu[2 * q]; v.y -= mu[2 * q + 1]; }
            const float w = win[j];
            fr[q * fst + j] = make_float2(v.x * w, v.y * w);
        }
        D4W_SYNC();
        fft_forward_stages(fr, wp.pl, wp.tw, npair, fst, tid, nthr, 0, wp.pl.nstages);
        for (int k = tid; k < nbins; k += nthr) {
            const int pk = wp.k2pos[k], pm = wp.k2pos[k == 0 ? 0 : n - k];
            const double f = (k == 0 || 2 * k == n) ? wp.scale : 2.0 * wp.scale;
            double acc = 0.0;
            for (int q = 0; q < npair; ++q) {
                const float2 z = fr[q * fst + pk], z2 = fr[q * fst + pm];
                const float ar = 0.5f * (z.x + z2.x), ai = 0.5f * (z.y - z2.y);
                const float br = 0.5f * (z.y + z2.y), bi = 0.5f * (z2.x - z.x);
                const double pa = (double)ar * ar + (double)ai * ai, pb = (double)br * br + (double)bi * bi;
                const bool has_b = 2 * q + 1 < cnt;
                if (wp.mode == kWelchMean) {
                    acc += pa;
                    if (has_b) acc += pb;
                } else {
                    const int s = s0 + 2 * q;
                    if (wp.mode == kWelchMedianSmem) {
                        per[(size_t)s * nbins + k] = (float)(pa * f);
                        if (has_b) per[(size_t)(s + 1) * nbins + k] = (float)(pb * f);
                    } else {
                        float* o = ws + ((size_t)block * nbins + k) * wp.nseg + s;
                        o[0] = (float)(pa * f);
                        if (has_b) o[1] = (float)(pb * f);
                    }
                }
            }
            if (wp.mode == kWelchMean) sums[k] += acc;
        }
        D4W_SYNC();                                                                 // frames are restaged next batch
    }
    float* o = out + (size_t)block * nbins;
    if (wp.mode == kWelchMean) {
        for (int k = tid; k < nbins; k += nthr) {
            const double f = (k == 0 || 2 * k == n) ? wp.scale : 2.0 * wp.scale;
            o[k] = (float)(sums[k] * f);
        }
    } else if (wp.mode == kWelchMedianSmem) {
        // exact np.median over the segments of each bin: v_i is order statistic r iff #{v < v_i} <= r < #{v <= v_i}
        const int rlo = (wp.nseg - 1) / 2, rhi = wp.nseg / 2;
        for (int k = tid; k < nbins; k += nthr) {
            float vlo = 0.f, vhi = 0.f;
            for (int i = 0; i < wp.nseg; ++i) {
                const float vi = per[(size_t)i * nbins + k];
                int lt = 0, le = 0;
                for (int j = 0; j < wp.nseg; ++j) {
                    const float vj = per[(size_t)j * nbins + k];
                    lt += vj < vi ? 1 : 0;
                    le += vj <= vi ? 1 : 0;
                }
                if (lt <= rlo && rlo < le) vlo = vi;
                if (lt <= rhi && rhi < le) vhi = vi;
            }
            o[k] = 0.5f * (vlo + vhi);
        }
    }
}

}  // namespace d4w
