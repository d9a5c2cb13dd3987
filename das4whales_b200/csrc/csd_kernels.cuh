// csd_kernels.cuh -- cross-spectral density and coherence of row pairs (d4w_csd, d4w_csd.cu): scipy.signal.csd and
// scipy.signal.coherence of output row r = (row r of x, row r of y), a row stride of 0 broadcasting one row.
//
// One CTA per output row.  Segment s is samples [s * step, s * step + nperseg), nseg = (ns - nperseg) / step + 1 (SciPy drops
// a trailing partial segment).  Segments go through the shared-memory FFT engine in batches of up to kCsdMaxFrames complex
// nfft-point frames, segment s of x in the real part and segment s of y in the imaginary part of one frame:
//   stage     frame q <- segment s0 + q of x (re) and of y (im), zero-padded to nfft
//   detrend   'constant': each half's own mean (double, fixed summation order) is subtracted, then the window multiplies
//   balance   each half is multiplied by the power of two 2^-e that brings its largest |value| into [0.5, 1), and the
//             products below by 2^(e_x + e_y) (exact both ways): x and y share one transform, and a row many orders of
//             magnitude below its partner (a strain row against a hydrophone in Pa) would otherwise drown in the
//             partner's float32 rounding
//   FFT       fft_forward_stages over the batch's frames
//   untangle  X_k = (Z_k + conj Z_{n-k}) / 2, Y_k = (Z_k - conj Z_{n-k}) / 2i at the one-sided bins k = 0 .. nfft/2, read at
//             k2pos[k] and k2pos[n - k] (the position map of the stages in `pl`, as welch_body reads it);
//             P_k = conj(X_k) Y_k times scale and SciPy's one-sided doubling (every bin but DC and, for even nfft, Nyquist)
//   average   mean: Re P and Im P (and, for the coherence, |X|^2 and |Y|^2) summed in double in segment order in shared
//             memory; the coherence |sum P|^2 / (sum |X|^2 sum |Y|^2) is divided in double and rounded once (0 / 0 is NaN,
//             as in NumPy);
//             median in shared memory (nseg <= kWelchSmemMedianSeg and every periodogram fits the budget): exact rank
//             selection per bin of Re and of Im, the two middle order statistics averaged for even nseg (np.median);
//             median through the workspace: periodograms written [row][bin][re|im][nseg], ws[((row * nbins + k) * 2 + c)
//             * nseg + s], then csd_median_body selects each row of nseg signed values; its output, one float per
//             (row, bin, re|im), is the interleaved complex result.
// For the median the periodograms are scaled by 1 / _median_bias(nseg) before the selection; the scaling is positive, so
// the selected order statistics are those of the unscaled values.
//
// The bodies are __host__ __device__ with (block, tid, nthr, smem) loops, so that tests/host_emul/csd_emul.cu runs them
// block by block on the CPU.
#pragma once
#include <cmath>
#include <cstring>
#include "welch_kernels.cuh"

namespace d4w {

enum { kCsdMean = 0, kCsdMedianSmem = 1, kCsdMedianWs = 2 };
// Frames per FFT batch.  Eight rather than four: the workspace route writes eight consecutive floats of each (bin, re|im)
// row per batch instead of four (whole 32-byte sectors only when nseg is a multiple of 8), and short frames make wider FFT
// batches; measured on an H100 in DESIGN.md §4
constexpr int kCsdMaxFrames = 8;

struct CsdParams {
    FftPlan pl;
    const float2* tw;
    const int* k2pos;            // DFT bin -> position after the forward stages of pl
    long long xstride, ystride;  // floats between rows of x / y; 0 broadcasts one row
    int nfft, nperseg, step, ns, nseg, nbins;
    int frames;                  // complex frames (segments of x and y) per batch
    int fstride;                 // float2 between frames (odd for even nfft)
    int detrend;                 // 1: subtract each segment's mean
    int coherence;               // 1: Cxy (mean only), else Pxy
    int mode;                    // kCsdMean / kCsdMedianSmem / kCsdMedianWs
    double scale;                // SciPy's scale, divided by nseg (mean) or by _median_bias(nseg) (median)
};

// bin sums of the mean route: Re P, Im P, and for the coherence |X|^2, |Y|^2
__host__ __device__ inline int csd_nsums(int coherence) { return coherence ? 4 : 2; }

// shared-memory layout of one CTA: [partial sums: kWelchThreads doubles][bin sums: csd_nsums x nbins doubles (mean)]
// [frames: frames x fstride float2][periodograms: 2 x nseg x nbins floats (median in shared memory)]
// [segment means, balance scales 2^-e and their inverses 2^e: 3 x 2 x kCsdMaxFrames floats]
__host__ __device__ inline size_t csd_smem_bytes(int nfft, int nbins, int nseg, int frames, int mode, int coherence) {
    return (size_t)kWelchThreads * sizeof(double) + (mode == kCsdMean ? (size_t)csd_nsums(coherence) * nbins * sizeof(double) : 0) +
           (size_t)frames * welch_fstride(nfft) * sizeof(float2) +
           (mode == kCsdMedianSmem ? (size_t)2 * nseg * nbins * sizeof(float) : 0) + (size_t)6 * kCsdMaxFrames * sizeof(float);
}

// Geometry, averaging route and batch size.  Returns 0, or 1 when one frame does not fit `smem_cap` (the nfft limit);
// `smem` is the CTA's shared memory.  Sizes must already be valid (d4w_csd checks them).
inline int csd_config(const FftPlan& pl, int ns, int nperseg, int step, int detrend, double scale, int coherence, int median,
                      size_t smem_cap, CsdParams& cp, size_t& smem) {
    cp = CsdParams{};
    cp.pl = pl;
    cp.nfft = pl.n; cp.nperseg = nperseg; cp.step = step; cp.ns = ns;
    cp.nseg = (ns - nperseg) / step + 1;
    cp.nbins = pl.n / 2 + 1;
    cp.fstride = welch_fstride(pl.n);
    cp.detrend = detrend ? 1 : 0;
    cp.coherence = coherence ? 1 : 0;
    cp.mode = !median ? kCsdMean
            : (cp.nseg <= kWelchSmemMedianSeg &&
               csd_smem_bytes(pl.n, cp.nbins, cp.nseg, 1, kCsdMedianSmem, 0) <= kWelchSmemBudget) ? kCsdMedianSmem
            : kCsdMedianWs;
    cp.scale = median ? scale / welch_median_bias(cp.nseg) : scale / cp.nseg;
    const int want = std::min(kCsdMaxFrames, cp.nseg);
    cp.frames = 1;
    while (cp.frames < want && csd_smem_bytes(pl.n, cp.nbins, cp.nseg, cp.frames + 1, cp.mode, cp.coherence) <= kWelchSmemBudget)
        ++cp.frames;
    smem = csd_smem_bytes(pl.n, cp.nbins, cp.nseg, cp.frames, cp.mode, cp.coherence);
    return smem <= smem_cap ? 0 : 1;
}

// One output row = `block`.  x, y: rows at x + block * xstride, y + block * ystride, ns samples each.  out: float2
// [nrows][nbins] (Pxy) or float [nrows][nbins] (Cxy); ws: the periodograms of kCsdMedianWs.
__host__ __device__ inline void csd_body(const CsdParams& cp, const float* __restrict__ x, const float* __restrict__ y,
                                         const float* __restrict__ win, void* __restrict__ out, float* __restrict__ ws,
                                         long long block, int tid, int nthr, void* smem) {
    const int n = cp.nfft, L = cp.nperseg, fst = cp.fstride, nbins = cp.nbins, nseg = cp.nseg;
    const int nsum = cp.mode == kCsdMean ? csd_nsums(cp.coherence) : 0;
    double* part = static_cast<double*>(smem);                                      // [kWelchThreads]
    double* sums = part + kWelchThreads;                                            // [nsum][nbins] (mean)
    float2* fr = reinterpret_cast<float2*>(sums + (size_t)nsum * nbins);
    float* per = reinterpret_cast<float*>(fr + (size_t)cp.frames * fst);           // [re|im][nseg][nbins] (median in smem)
    float* mu = per + (cp.mode == kCsdMedianSmem ? (size_t)2 * nseg * nbins : 0);  // [2 * kCsdMaxFrames]
    float* sc = mu + 2 * kCsdMaxFrames;                                            // 2^-e per half
    float* un = sc + 2 * kCsdMaxFrames;                                            // 2^e per half
    const float* xr = x + block * cp.xstride;
    const float* yr = y + block * cp.ystride;
    const int halves = 2 * cp.frames;
    const int G = nthr / halves > 0 ? nthr / halves : 1;                            // partial sums per segment mean
    for (int i = tid; i < nsum * nbins; i += nthr) sums[i] = 0.0;
    for (int s0 = 0; s0 < nseg; s0 += cp.frames) {
        const int cnt = nseg - s0 < cp.frames ? nseg - s0 : cp.frames;              // frames in this batch
        for (int i = tid; i < cnt * n; i += nthr) {
            const int q = i / n, j = i - q * n;
            float a = 0.f, b = 0.f;
            if (j < L) {
                a = xr[(size_t)(s0 + q) * cp.step + j];
                b = yr[(size_t)(s0 + q) * cp.step + j];
            }
            fr[q * fst + j] = make_float2(a, b);
        }
        D4W_SYNC();
        if (cp.detrend) {
            for (int id = tid; id < halves * G; id += nthr) {
                const int h = id / G, l = id - h * G;
                double acc = 0.0;
                if ((h >> 1) < cnt) {
                    const float* f = reinterpret_cast<const float*>(fr + (size_t)(h >> 1) * fst) + (h & 1);
                    for (int j = l; j < L; j += G) acc += (double)f[2 * j];
                }
                part[id] = acc;
            }
            D4W_SYNC();
            for (int h = tid; h < halves; h += nthr) {
                double acc = 0.0;
                for (int l = 0; l < G; ++l) acc += part[h * G + l];
                mu[h] = (h >> 1) < cnt ? (float)(acc / L) : 0.f;
            }
            D4W_SYNC();
        }
        for (int id = tid; id < halves * G; id += nthr) {                           // balance: largest |value| per half
            const int h = id / G, l = id - h * G;
            float m = 0.f;
            if ((h >> 1) < cnt) {
                const float* f = reinterpret_cast<const float*>(fr + (size_t)(h >> 1) * fst) + (h & 1);
                const float c = cp.detrend ? mu[h] : 0.f;
                for (int j = l; j < L; j += G) m = fmaxf(m, fabsf((f[2 * j] - c) * win[j]));
            }
            part[id] = m;
        }
        D4W_SYNC();
        for (int h = tid; h < halves; h += nthr) {
            double m = 0.0;
            for (int l = 0; l < G; ++l) m = fmax(m, part[h * G + l]);
            int e = 0;
            if (m > 0.0) frexp(m, &e);
            e = e < -126 ? -126 : e > 126 ? 126 : e;                                // 2^-e and 2^e stay normal floats
            sc[h] = ldexpf(1.f, -e);
            un[h] = m > 0.0 ? ldexpf(1.f, e) : 0.f;     // an all-zero half adds exact zeros, not its partner's rounding
        }
        D4W_SYNC();
        for (int i = tid; i < cnt * L; i += nthr) {
            const int q = i / L, j = i - q * L;
            float2 v = fr[q * fst + j];
            if (cp.detrend) { v.x -= mu[2 * q]; v.y -= mu[2 * q + 1]; }
            const float w = win[j];
            fr[q * fst + j] = make_float2(v.x * w * sc[2 * q], v.y * w * sc[2 * q + 1]);
        }
        D4W_SYNC();
        fft_forward_stages(fr, cp.pl, cp.tw, cnt, fst, tid, nthr, 0, cp.pl.nstages);
        for (int k = tid; k < nbins; k += nthr) {
            const int pk = cp.k2pos[k], pm = cp.k2pos[k == 0 ? 0 : n - k];
            const double f = (k == 0 || 2 * k == n) ? cp.scale : 2.0 * cp.scale;
            double are = 0.0, aim = 0.0, axx = 0.0, ayy = 0.0;
            for (int q = 0; q < cnt; ++q) {
                const float2 z = fr[q * fst + pk], z2 = fr[q * fst + pm];
                const float ar = 0.5f * (z.x + z2.x), ai = 0.5f * (z.y - z2.y);      // X_k
                const float br = 0.5f * (z.y + z2.y), bi = 0.5f * (z2.x - z.x);      // Y_k
                const double ux = un[2 * q], uy = un[2 * q + 1], uxy = ux * uy;          // undo the balance
                const double re = ((double)ar * br + (double)ai * bi) * uxy, im = ((double)ar * bi - (double)ai * br) * uxy;
                if (cp.mode == kCsdMean) {
                    are += re;
                    aim += im;
                    if (cp.coherence) {
                        axx += ((double)ar * ar + (double)ai * ai) * (ux * ux);
                        ayy += ((double)br * br + (double)bi * bi) * (uy * uy);
                    }
                } else if (cp.mode == kCsdMedianSmem) {
                    per[(size_t)(s0 + q) * nbins + k] = (float)(re * f);
                    per[(size_t)(nseg + s0 + q) * nbins + k] = (float)(im * f);
                } else {
                    float* o = ws + ((size_t)block * nbins + k) * 2 * nseg + s0 + q;
                    o[0] = (float)(re * f);
                    o[nseg] = (float)(im * f);
                }
            }
            if (cp.mode == kCsdMean) {
                sums[k] += are;
                sums[nbins + k] += aim;
                if (cp.coherence) { sums[2 * nbins + k] += axx; sums[3 * nbins + k] += ayy; }
            }
        }
        D4W_SYNC();                                                                 // frames are restaged next batch
    }
    if (cp.mode == kCsdMean && cp.coherence) {
        float* o = static_cast<float*>(out) + (size_t)block * nbins;
        for (int k = tid; k < nbins; k += nthr) {
            const double re = sums[k], im = sums[nbins + k];
            o[k] = (float)((re * re + im * im) / (sums[2 * nbins + k] * sums[3 * nbins + k]));
        }
    } else if (cp.mode == kCsdMean) {
        float2* o = static_cast<float2*>(out) + (size_t)block * nbins;
        for (int k = tid; k < nbins; k += nthr) {
            const double f = (k == 0 || 2 * k == n) ? cp.scale : 2.0 * cp.scale;
            o[k] = make_float2((float)(sums[k] * f), (float)(sums[nbins + k] * f));
        }
    } else if (cp.mode == kCsdMedianSmem) {
        // exact np.median over the segments of each bin: v_i is order statistic r iff #{v < v_i} <= r < #{v <= v_i}
        float* o = static_cast<float*>(out) + (size_t)block * nbins * 2;
        const int rlo = (nseg - 1) / 2, rhi = nseg / 2;
        for (int i = tid; i < 2 * nbins; i += nthr) {
            const int k = i >> 1, c = i & 1;
            const float* v = per + (size_t)c * nseg * nbins + k;
            float vlo = 0.f, vhi = 0.f;
            for (int a = 0; a < nseg; ++a) {
                const float va = v[(size_t)a * nbins];
                int lt = 0, le = 0;
                for (int b = 0; b < nseg; ++b) {
                    const float vb = v[(size_t)b * nbins];
                    lt += vb < va ? 1 : 0;
                    le += vb <= va ? 1 : 0;
                }
                if (lt <= rlo && rlo < le) vlo = va;
                if (lt <= rhi && rhi < le) vhi = va;
            }
            o[i] = 0.5f * (vlo + vhi);
        }
    }
}

// ---- exact np.median of rows of signed floats (the workspace route): a radix selection on order-preserving keys
// One row per group of G = min(nthr, 32) threads (a warp on the GPU; G = nthr = 1 on the host), rows block * (nthr / G) + g.
// Each order statistic takes four passes over the row, one per key byte from the top: a 256-bin histogram of the rows'
// values that share the key prefix chosen so far, then the bin that holds the wanted rank.  The result is exact: the
// two middle order statistics (one for odd n) are averaged as np.median averages them.  nthr must be a power of two.
constexpr int kCsdSelThreads = 256;
constexpr int kCsdSelGroup = 32;
constexpr int kCsdSelInts = 256 + kCsdSelGroup + 2;  // shared ints per group: histogram, lane sums, chosen bin and rank

// Keys whose unsigned order is the order of the floats (-0 sorts just below +0; there are no NaNs in a periodogram).
__host__ __device__ inline unsigned csd_key(float v) {
    unsigned u;
#ifdef __CUDA_ARCH__
    u = __float_as_uint(v);
#else
    std::memcpy(&u, &v, sizeof u);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__host__ __device__ inline float csd_unkey(unsigned k) {
    const unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float v;
    std::memcpy(&v, &u, sizeof v);
    return v;
#endif
}

__host__ __device__ inline void csd_median_body(const float* __restrict__ v, long long nrows, int n, float* __restrict__ out,
                                                long long block, int tid, int nthr, void* smem) {
    const int G = nthr < kCsdSelGroup ? nthr : kCsdSelGroup;
    const int g = tid / G, lane = tid - g * G, per = 256 / G;
    const long long row = block * (nthr / G) + g;
    const bool active = row < nrows;
    int* hist = static_cast<int*>(smem) + (size_t)g * kCsdSelInts;
    int* lsum = hist + 256;
    int* sel = lsum + kCsdSelGroup;
    const float* r = v + (size_t)(active ? row : 0) * n;
    float res[2] = {0.f, 0.f};
    for (int h = 0; h < 2; ++h) {
        if (h == 1 && n % 2 == 1) { res[1] = res[0]; break; }                       // odd n: one middle value
        unsigned prefix = 0;
        int rank = h == 0 ? (n - 1) / 2 : n / 2;                                    // rank among the values with the prefix
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int b = lane; b < 256; b += G) hist[b] = 0;
            D4W_SYNC();
            if (active)
                for (int i = lane; i < n; i += G) {
                    const unsigned key = csd_key(r[i]);
                    if (shift == 24 || (key >> (shift + 8)) == (prefix >> (shift + 8))) {
#ifdef __CUDA_ARCH__
                        atomicAdd(&hist[(key >> shift) & 255u], 1);
#else
                        ++hist[(key >> shift) & 255u];
#endif
                    }
                }
            D4W_SYNC();
            int s = 0;
            for (int b = lane * per; b < (lane + 1) * per; ++b) s += hist[b];
            lsum[lane] = s;
            D4W_SYNC();
            int c = 0;
            for (int l = 0; l < lane; ++l) c += lsum[l];
            if (c <= rank && rank < c + s) {                                        // one lane per active group
                int b = lane * per;
                while (c + hist[b] <= rank) c += hist[b++];
                sel[0] = b;
                sel[1] = rank - c;
            }
            D4W_SYNC();
            prefix |= (unsigned)sel[0] << shift;
            rank = sel[1];
        }
        res[h] = csd_unkey(prefix);
    }
    if (active && lane == 0) out[row] = 0.5f * (res[0] + res[1]);
}

}  // namespace d4w
