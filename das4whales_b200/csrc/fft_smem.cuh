// fft_smem.cuh -- shared-memory mixed-radix FFT engine (in place, self-sorting by pairing).
//
// A length-N transform is a sequence of radix stages.  The forward transform is
// decimation-in-frequency: natural order in, digit-reversed order out; every butterfly
// reads and writes the SAME R shared-memory words, so a stage needs one __syncthreads and
// no second buffer (a 10 000-point complex column pair already fills 160 KB of the 227 KB).
// The inverse transform is the exact mirror (decimation-in-time, digit-reversed in, natural
// out), so  forward -> pointwise multiply -> inverse  never needs a reordering pass: the
// multiplier table is simply stored in digit-reversed order (fk mask, Hilbert weights,
// matched-filter template spectrum all use this).
//
// Twiddles: one table W_N^j (fp32, rounded once from double on the host) per length; a stage
// fetches W_Ns^n = tab[(N/Ns)*n] and forms the R-1 powers by a balanced product tree.
// Prime factors 7..61 run through a generic O(p^2) stage (OOI channel counts are 2*5*19*29).
#pragma once
#include "fft_radix.cuh"

namespace d4w {

constexpr int kMaxStages = 12;

struct FftPlan {
    int n;                    // transform length
    int nstages;
    int radix[kMaxStages];    // forward (DIF) stage order
    int sub[kMaxStages];      // sub-transform length entering stage s (sub[0] = n)
};

#ifdef __CUDA_ARCH__
#define D4W_SYNC() __syncthreads()
#else
#define D4W_SYNC() ((void)0)
#endif

// ---- one in-place radix-R stage over `nfft` transforms stored `fstride` apart -----------
// DIF (forward):  v[m] = (sum_q u[q] W_R^{qm}) * W_Ns^{n m};   DIT (inverse) undoes exactly that.
template <int R, bool INV>
__host__ __device__ void stage_inreg(float2* __restrict__ s, const float2* __restrict__ tw, int n_total,
                                     int ns, int nfft, int fstride, int tid, int nthr) {
    const int L = ns / R;                 // butterfly leg spacing
    const int per = n_total / R;          // butterflies per transform
    const int twstep = n_total / ns;      // tab stride for W_Ns
    const int total = per * nfft;
    // many small transforms (STFT frames): make the transform index the fast lane index so that, with an odd
    // fstride, neighbouring lanes fall into different banks even in the short-stride last stages
    const bool f_fast = nfft >= 16;
    for (int id = tid; id < total; id += nthr) {
        const int f = f_fast ? id % nfft : id / per;
        const int j = f_fast ? id / nfft : id - f * per;
        const int b = j / L;
        const int n = j - b * L;
        float2* base = s + (size_t)f * fstride + b * ns + n;
        float2 v[R];
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; v[q] = base[q * L]; });
        if constexpr (!INV) {
            DFT<R, false>::run(v);
            if (L > 1) {
                float2 p[R];
                twiddle_powers<R>(tw[twstep * n], p);
                static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; if constexpr (m > 0) v[m] = cmul(v[m], p[m]); });
            }
        } else {
            if (L > 1) {
                float2 p[R];
                twiddle_powers<R>(tw[twstep * n], p);
                static_for<R>([&](auto mc) { constexpr int m = decltype(mc)::value; if constexpr (m > 0) v[m] = cmulc(v[m], p[m]); });
            }
            DFT<R, true>::run(v);
        }
        static_for<R>([&](auto qc) { constexpr int q = decltype(qc)::value; base[q * L] = v[q]; });
    }
}

// ---- generic prime-radix stage (7 <= p <= 61): one thread per output element -------------
// Butterfly outputs overwrite inputs other lanes still need, so work is cut into chunks of
// whole butterflies: compute into a register, barrier, write, barrier.
template <bool INV>
__host__ __device__ void stage_generic(float2* __restrict__ s, const float2* __restrict__ tw, int n_total,
                                       int ns, int p, int nfft, int fstride, int tid, int nthr) {
    const int L = ns / p;
    const int per = n_total / p;
    const int twstep = n_total / ns;
    const int twp = n_total / p;                 // tab stride for W_p
    const int total = per * nfft;
#ifdef __CUDA_ARCH__
    const int bpc = nthr / p;                    // butterflies per chunk
    for (int c0 = 0; c0 < total; c0 += bpc) {
        const int id = c0 + tid / p;
        const int m = tid % p;
        const bool act = (tid < bpc * p) && (id < total);
        float2 acc = make_float2(0.f, 0.f);
        float2* base = s;
        if (act) {
            const int f = id / per, j = id - f * per, b = j / L, n = j - b * L;
            base = s + (size_t)f * fstride + b * ns + n;
            if (!INV) {
                for (int q = 0; q < p; ++q) acc = cadd(acc, cmul(base[q * L], tw[twp * ((q * m) % p)]));
                if (L > 1) acc = cmul(acc, tw[(int)(((long long)twstep * n * m) % n_total)]);
            } else {
                for (int q = 0; q < p; ++q) {
                    float2 u = base[q * L];
                    if (L > 1) u = cmulc(u, tw[(int)(((long long)twstep * n * q) % n_total)]);
                    acc = cadd(acc, cmulc(u, tw[twp * ((q * m) % p)]));
                }
            }
        }
        __syncthreads();
        if (act) base[m * L] = acc;
        __syncthreads();
    }
#else
    // host emulation: sequential, one butterfly at a time with a local copy
    if (tid != 0) return;
    for (int id = 0; id < total; ++id) {
        const int f = id / per, j = id - f * per, b = j / L, n = j - b * L;
        float2* base = s + (size_t)f * fstride + b * ns + n;
        float2 in[64], out[64];
        for (int q = 0; q < p; ++q) in[q] = base[q * L];
        for (int m = 0; m < p; ++m) {
            float2 acc = make_float2(0.f, 0.f);
            if (!INV) {
                for (int q = 0; q < p; ++q) acc = cadd(acc, cmul(in[q], tw[twp * ((q * m) % p)]));
                if (L > 1) acc = cmul(acc, tw[(int)(((long long)twstep * n * m) % n_total)]);
            } else {
                for (int q = 0; q < p; ++q) {
                    float2 u = in[q];
                    if (L > 1) u = cmulc(u, tw[(int)(((long long)twstep * n * q) % n_total)]);
                    acc = cadd(acc, cmulc(u, tw[twp * ((q * m) % p)]));
                }
            }
            out[m] = acc;
        }
        for (int m = 0; m < p; ++m) base[m * L] = out[m];
    }
#endif
}

template <bool INV>
__host__ __device__ inline void stage_dispatch(float2* s, const float2* tw, int n_total, int ns, int r,
                                               int nfft, int fstride, int tid, int nthr) {
    switch (r) {
#define D4W_CASE(RR) case RR: stage_inreg<RR, INV>(s, tw, n_total, ns, nfft, fstride, tid, nthr); break;
        D4W_CASE(2) D4W_CASE(3) D4W_CASE(4) D4W_CASE(5) D4W_CASE(6) D4W_CASE(8) D4W_CASE(10)
        D4W_CASE(12) D4W_CASE(15) D4W_CASE(16) D4W_CASE(20) D4W_CASE(25)
#undef D4W_CASE
        default: stage_generic<INV>(s, tw, n_total, ns, r, nfft, fstride, tid, nthr); break;
    }
}

// Stages [s0, s1) of the forward transform (natural -> digit-reversed).  Caller must have
// synchronised after filling `s`; returns synchronised.
__host__ __device__ inline void fft_forward_stages(float2* s, const FftPlan& pl, const float2* tw, int nfft,
                                                   int fstride, int tid, int nthr, int s0, int s1) {
    for (int st = s0; st < s1; ++st) {
        stage_dispatch<false>(s, tw, pl.n, pl.sub[st], pl.radix[st], nfft, fstride, tid, nthr);
        D4W_SYNC();
    }
}
// Stages (s1, s0] of the inverse transform, i.e. undoing forward stages s1-1 ... s0.
__host__ __device__ inline void fft_inverse_stages(float2* s, const FftPlan& pl, const float2* tw, int nfft,
                                                   int fstride, int tid, int nthr, int s0, int s1) {
    for (int st = s1 - 1; st >= s0; --st) {
        stage_dispatch<true>(s, tw, pl.n, pl.sub[st], pl.radix[st], nfft, fstride, tid, nthr);
        D4W_SYNC();
    }
}

// (first, last) radix of every row plan whose middle pass runs as k_row_mid_fused: one kernel per pair, so each holds
// only its own butterflies (a run-time choice among all in-register radices spills at 128 registers).  The pairs are
// those build_fk_hostplan gives split rows (T1 > 1) of every 2^a 3^b 5^c length up to 25 x 10 240 -- every f-k,
// Hilbert and chirp-z row length with an in-register first and last stage; tests/test_row_fused_host.py re-derives
// the list from the planner.  A plan whose pair is not listed uses k_row_mid.
#define D4W_ROW_FUSED_PAIRS(X)                                                                                    \
    X(3, 3) X(6, 3) X(6, 5) X(6, 15) X(8, 15) X(10, 15) X(10, 25) X(12, 3) X(12, 5) X(15, 3) X(16, 3) X(16, 5)   \
    X(16, 8) X(16, 25) X(20, 15) X(20, 25) X(25, 5) X(25, 15)

// f(integral_constant R0, integral_constant RL) for a listed pair; false (f not called) for any other
template <class F>
__host__ __device__ inline bool with_row_fused_pair(int r0, int rl, F&& f) {
#define D4W_PAIR(A, B)                                                                        \
    if (r0 == A && rl == B) { f(std::integral_constant<int, A>{}, std::integral_constant<int, B>{}); return true; }
    D4W_ROW_FUSED_PAIRS(D4W_PAIR)
#undef D4W_PAIR
    return false;
}

// position -> frequency index after the forward transform (host side table builder)
inline int pos_to_freq(const FftPlan& pl, int p) {
    int k = 0, mult = 1, rem = p, len = pl.n;
    for (int s = 0; s < pl.nstages; ++s) {
        const int L = len / pl.radix[s];
        const int m = rem / L;
        rem -= m * L;
        k += m * mult;
        mult *= pl.radix[s];
        len = L;
    }
    return k;
}

}  // namespace d4w
